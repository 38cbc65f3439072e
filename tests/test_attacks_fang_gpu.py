"""fang-krum and fang-trim on sm_90a: the crafting kernels against the torch reference (fang-trim's rows bit for bit; fang-krum's gamma from
the kernel's own sums with the reference search, the sums against float64 statistics, the rows bit for bit), the fused engine against the
baseline engine through training, and the sharded crafting passes on several GPUs."""

import json
import math
import os
import pathlib
import subprocess
import sys

import pytest
import torch

from aggregathor_b200 import aggregators, attacks, experiments
from aggregathor_b200.aggregators import _ops
from aggregathor_b200.engine.trainer import Manager

pytestmark = pytest.mark.gpu
ROOT = pathlib.Path(__file__).resolve().parent.parent


def _bits(t):
  return t.detach().cpu().contiguous().view(torch.int32)


def _equal_values(a, b):
  """Equal bit for bit, except that any NaN matches any NaN (same positions)."""
  a, b = a.cpu(), b.cpu()
  nan = torch.isnan(a)
  assert torch.equal(nan, torch.isnan(b))
  assert torch.equal(_bits(a)[~nan], _bits(b)[~nan])


def _matrix(n, d, seed, honest=None):
  """Seeded rows over four decades around a common direction, zero columns; with `honest` slots, NaN, +inf and -inf go into three of them."""
  gen = torch.Generator().manual_seed(seed)
  G = (torch.randn(1, d, generator=gen) + 0.5 * torch.randn(n, d, generator=gen)) * torch.logspace(-2, 2, d)
  G[:, 11::97] = 0.0
  if honest is not None:
    G[honest[0], 3::101] = float("nan")
    G[honest[1 % len(honest)], 5::103] = float("inf")
    G[honest[-1], 7::107] = float("-inf")
  return G


def _trim_cases():
  for n in (3, 8, 9, 17, 32):
    for k in sorted({1, max(1, n // 3), n - 1}):
      yield n, k


@pytest.mark.parametrize("d", [200003, 200000])
@pytest.mark.parametrize("n,k", list(_trim_cases()))
def test_trim_kernel_matches_the_reference(n, k, d):
  from aggregathor_b200.ops import gar as gar_ops
  for first in (False, True):
    for non_finite in (False, True):
      byz = list(range(k)) if first else list(range(n - k, n))
      honest = [i for i in range(n) if i not in byz]
      G = _matrix(n, d, seed=n * 31 + k + d + first, honest=honest if non_finite else None)
      Gd = G.cuda()
      gar_ops.craft_byzantine_(Gd, byz, "fang-trim", scale=3.0, seed=7, step=12)
      torch.cuda.synchronize()
      expected = _ops.torch_craft_byzantine_(G.clone(), byz, "fang-trim", scale=3.0, seed=7, step=12)
      for i in range(n):
        if i in byz:
          _equal_values(Gd[i], expected[i])
        else:
          assert torch.equal(_bits(Gd[i]), _bits(G[i])), i   # honest rows byte-identical


def _krum_cases():
  for n in (4, 8, 9, 17, 32):
    for k in sorted({1, max(1, n // 4), (n - 2) // 2}):
      if n - 2 * k - 1 >= 1:
        yield n, k


def _check_krum_kernel(G, byz, f, non_finite):
  from aggregathor_b200.ops import gar as gar_ops
  n = G.shape[0]
  Gd = G.cuda()
  gamma, selected, t, gamma_max, A, B, C, T = gar_ops.craft_byzantine_(Gd, byz, "fang-krum", f=f, return_details=True)
  torch.cuda.synchronize()
  # the kernel searches from its own sums with exactly the reference's operations
  assert (gamma, selected, t, gamma_max) == _ops.fang_krum_gamma(A, B, C, T, n, f, byz, _ops.FANG_THRESHOLD)
  if non_finite:
    assert (gamma, selected, t) == (0.0, False, -1)
  else:
    # the fp32 sums against the float64 statistics (B within 1e-5 of its Cauchy-Schwarz bound sqrt(A_i C))
    _, _, A64, B64, C64, T64 = _ops.fang_krum_statistics(G.cuda(), byz)
    assert abs(C - C64) <= 1e-5 * C64
    for a, a64, b, b64 in zip(A, A64, B, B64):
      assert abs(a - a64) <= 1e-5 * a64 and abs(b - b64) <= 1e-5 * math.sqrt(a64 * C64), (a, a64, b, b64)
    for x, x64 in zip(T, T64):
      assert abs(x - x64) <= 1e-5 * x64
    assert gamma > 0 and t >= 0
  honest = [G[i] for i in range(n) if i not in byz]
  row = torch.neg(torch.tensor(gamma)) * _ops._sign(_ops._honest_mean(honest, _ops._scalar(G)))
  for i in range(n):
    if i in byz:
      _equal_values(Gd[i], row)
    else:
      assert torch.equal(_bits(Gd[i]), _bits(G[i])), i


@pytest.mark.parametrize("d", [200003, 200000])
@pytest.mark.parametrize("n,k", list(_krum_cases()))
def test_krum_kernel_matches_the_reference(n, k, d):
  for first in (False, True):
    for non_finite in (False, True):
      byz = list(range(k)) if first else list(range(n - k, n))
      honest = [i for i in range(n) if i not in byz]
      G = _matrix(n, d, seed=n * 37 + k + d + first, honest=honest if non_finite else None)
      _check_krum_kernel(G, byz, min(k, n - 3), non_finite)


def test_krum_kernel_selection_is_effective():
  """Independent standard normal rows, four Byzantine rows out of 17: the search stops at a selected candidate, and Krum on the crafted
  rows picks a Byzantine one."""
  from aggregathor_b200.ops import gar as gar_ops
  gen = torch.Generator().manual_seed(3)
  G = torch.randn(17, 4001, generator=gen)
  Gd = G.cuda()
  gamma, selected, t, gamma_max, A, B, C, T = gar_ops.craft_byzantine_(Gd, [13, 14, 15, 16], "fang-krum", f=4, return_details=True)
  assert (gamma, selected, t, gamma_max) == _ops.fang_krum_gamma(A, B, C, T, 17, 4, [13, 14, 15, 16], _ops.FANG_THRESHOLD)
  assert selected and gamma > 0
  _, chosen = _ops.torch_krum(Gd.cpu(), 4, 1, return_selected=True)
  assert int(chosen[0]) in (13, 14, 15, 16)


def test_krum_kernel_without_the_search_returns_gamma_max():
  from aggregathor_b200.ops import gar as gar_ops
  G = _matrix(8, 4000, seed=9).cuda()
  launcher = gar_ops._launcher(G.device, 8)
  rows = [G.data_ptr() + i * 4000 * 4 for i in range(8)]
  gar_ops.craft(rows, [(0, 4000)], list(range(6)), [6, 7], "fang-krum", None, f=2, launcher=launcher, search=False)
  gamma, selected, t, gamma_max, *_ = gar_ops.fang_krum_details(launcher, 6)
  assert not selected and t == 0 and gamma == _ops.fp32(gamma_max) and gamma > 0


def test_kernels_leave_a_strided_caller_matrix_alone_outside_the_byzantine_rows():
  from aggregathor_b200.ops import gar as gar_ops
  base = torch.randn(9, 1030, device="cuda")
  before = base.clone()
  G = base[:, 3:1004]   # not contiguous, not 16-byte aligned: crafted on a padded copy, written back
  gamma, *_ = gar_ops.craft_byzantine_(G, [7, 8], "fang-krum", f=2, return_details=True)
  ref = before[:, 3:1004].cpu().contiguous()
  expected = torch.neg(torch.tensor(gamma)) * _ops._sign(_ops._honest_mean(list(ref[:7]), _ops._scalar(ref)))
  _equal_values(G[7], expected)
  _equal_values(G[8], expected)
  assert torch.equal(base[:7], before[:7]) and torch.equal(base[:, :3], before[:, :3]) and torch.equal(base[:, 1004:], before[:, 1004:])
  gar_ops.craft_byzantine_(G, [7, 8], "fang-trim", seed=1, step=2)
  expected = _ops.torch_craft_byzantine_(ref.clone(), [7, 8], "fang-trim", seed=1, step=2)
  _equal_values(G[7], expected[7])
  _equal_values(G[8], expected[8])
  assert torch.equal(base[:7], before[:7]) and torch.equal(base[:, :3], before[:, :3]) and torch.equal(base[:, 1004:], before[:, 1004:])


def test_more_than_32_workers_use_the_torch_reference():
  from aggregathor_b200.ops import gar as gar_ops
  G = torch.randn(36, 999, generator=torch.Generator().manual_seed(8))
  Gd = G.cuda()
  details = gar_ops.craft_byzantine_(Gd, [33, 34, 35], "fang-krum", f=3, return_details=True)
  assert len(details[4]) == 33 and details[:4] == _ops.fang_krum_gamma(*details[4:], 36, 3, [33, 34, 35], _ops.FANG_THRESHOLD)
  Gd = G.cuda()
  gar_ops.craft_byzantine_(Gd, [0, 35], "fang-trim", step=4)
  expected = _ops.torch_craft_byzantine_(G.clone(), [0, 35], "fang-trim", step=4)
  _equal_values(Gd[0], expected[0])
  _equal_values(Gd[35], expected[35])


def _manager(rule, n, k, mode, engine):
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate(rule, n, k, [])
  return Manager(experiment, gar, n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cuda", engine=engine, seed=7,
                 attack=attacks.instantiate(mode, n, k, ["seed:3"] if mode == "fang-trim" else []), nb_real_byz=k)


@pytest.mark.parametrize("mode", ["fang-krum", "fang-trim"])
@pytest.mark.parametrize("rule", ["krum", "trimmed-mean", "median"])
def test_fused_engine_matches_the_baseline_engine(rule, mode):
  """Both engines run the crafting kernels at R = 1 on the same owned coordinates [0, d): same grid, same fold order, same bits."""
  n = 11
  fused = _manager(rule, n, 2, mode, "fused")
  base = _manager(rule, n, 2, mode, "baseline")
  assert fused.aggregation.name == "fused" and base.aggregation.name == "baseline"
  for _ in range(3):
    fused.train()
    base.train()
    torch.cuda.synchronize()
    assert fused.aggregation.last_craft == base.aggregation.last_craft
    if mode == "fang-krum":
      assert fused.aggregation.last_craft[0] > 0
    for i in (n - 2, n - 1):
      assert torch.equal(_bits(fused.aggregation.visible_rows()[i]), _bits(base.aggregation.visible_rows()[i]))
  assert torch.equal(_bits(fused.params), _bits(base.params))
  fused.close()
  base.close()


def _gpus():
  return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_gpus() < 2, reason="needs at least 2 GPUs")
@pytest.mark.parametrize("mode", ["fang-krum", "fang-trim"])
def test_sharded_crafting_on_several_gpus(tmp_path, mode):
  """n = 8 over 2 or 4 ranks, both Byzantine workers on the last rank: fang-krum solves the same gamma on every rank and crafts the
  reference row for it; fang-trim's rows are the baseline engine's, bit for bit."""
  nproc = 4 if _gpus() >= 4 else 2
  port = 29900 + os.getpid() % 90
  cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1", "--master-port", str(port),
         str(ROOT / "benchmarks" / "gar_bench.py"), "--gar-dim", "1000003", "--gar-iters", "3", "--gar-rules", "krum,trimmed-mean", "--gar-out", str(tmp_path),
         "--gar-attack", mode, "--gar-dump-rows"]
  proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, cwd=str(ROOT))
  out = proc.stdout.decode(errors="replace")
  assert proc.returncode == 0, out[-4000:]
  results = json.loads((tmp_path / ("gar_bench_%d.json" % nproc)).read_text())["results"]
  for rule in ("krum", "trimmed-mean"):
    entry = results[rule]
    assert entry["attack"] == mode and entry["replicas_identical"], (rule, entry)
    dump = torch.load(tmp_path / ("gar_rows_%s_%d.pt" % (rule, nproc)))
    rows, byz = dump["rows"], dump["byzantine"]
    assert byz == [6, 7]
    if mode == "fang-krum":
      gammas = entry["gamma_per_rank"]
      assert len(gammas) == nproc and len(set(gammas)) == 1 and gammas[0] > 0 and dump["gamma"] == gammas[0], (rule, entry)
      expected = torch.neg(torch.tensor(gammas[0])) * _ops._sign(_ops._honest_mean(list(rows[:6]), _ops._scalar(rows)))
      for i in byz:
        _equal_values(rows[i], expected)
    else:
      assert entry["rows_match_baseline"], (rule, entry)

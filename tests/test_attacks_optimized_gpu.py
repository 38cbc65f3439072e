"""Min-Max and Min-Sum on sm_90a: the crafting kernel against the torch reference (gamma against the float64 statistics, the rows bit for
bit for the kernel's own gamma), the fused engine against the baseline engine through training, and the sharded crafting pass with its
cross-rank exchange on several GPUs."""

import json
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
MODES = ("min-max", "min-sum")
DEVIATIONS = ("unit-vec", "sign", "std")


def _bits(t):
  return t.detach().cpu().contiguous().view(torch.int32)


def _equal_values(a, b):
  """Equal bit for bit, except that any NaN matches any NaN (same positions)."""
  a, b = a.cpu(), b.cpu()
  nan = torch.isnan(a)
  assert torch.equal(nan, torch.isnan(b))
  assert torch.equal(_bits(a)[~nan], _bits(b)[~nan])


def _matrix(n, d, seed, honest=None):
  """Seeded rows over four decades around a common direction; with `honest` slots, NaN, +inf and -inf go into three of them."""
  gen = torch.Generator().manual_seed(seed)
  G = (torch.randn(1, d, generator=gen) + 0.5 * torch.randn(n, d, generator=gen)) * torch.logspace(-2, 2, d)
  if honest is not None:
    G[honest[0], 3::101] = float("nan")
    G[honest[1 % len(honest)], 5::103] = float("inf")
    G[honest[-1], 7::107] = float("-inf")
  return G


def _cases():
  for n in (3, 8, 9, 17, 32):
    for k in sorted({1, max(1, n // 3), n - 2}):
      yield n, k


def _check_kernel(G, byz, mode, deviation, non_finite):
  from aggregathor_b200.ops import gar as gar_ops
  n = G.shape[0]
  Gd = G.cuda()
  gamma, A, B, C, T = gar_ops.craft_byzantine_(Gd, byz, mode, deviation=deviation, return_details=True)
  torch.cuda.synchronize()
  # the kernel solves gamma from its own sums with exactly the reference solver's operations
  assert gamma == _ops.optimized_gamma(mode, A, B, C, T), (mode, deviation)
  # against the float64 statistics of the reference (the sums taken in float64 on the device)
  _, _, A64, B64, C64, T64 = _ops.optimized_statistics(G.cuda(), byz, mode, deviation)
  expected_gamma = _ops.optimized_gamma(mode, A64, B64, C64, T64)
  if non_finite:
    assert gamma == 0.0 == expected_gamma
  else:
    assert gamma > 0 and abs(gamma - expected_gamma) <= 1e-5 * expected_gamma, (mode, deviation, gamma, expected_gamma)
  row = _ops.torch_optimized_row(G, byz, mode, deviation, gamma)   # CPU, the kernel's gamma
  for i in range(n):
    if i in byz:
      _equal_values(Gd[i], row)
    else:
      assert torch.equal(_bits(Gd[i]), _bits(G[i])), i   # honest rows byte-identical


@pytest.mark.parametrize("d", [400003, 400000])
@pytest.mark.parametrize("n,k", list(_cases()))
def test_kernel_matches_the_reference(n, k, d):
  for mode in MODES:
    for deviation in DEVIATIONS:
      for non_finite in (False, True):
        byz = list(range(n - k, n)) if mode == "min-max" else list(range(k))   # the Byzantine slots may come first too
        honest = [i for i in range(n) if i not in byz]
        G = _matrix(n, d, seed=n * 31 + k + d + len(deviation), honest=honest if non_finite else None)
        _check_kernel(G, byz, mode, deviation, non_finite)


def test_kernel_leaves_a_strided_caller_matrix_alone_outside_the_byzantine_rows():
  from aggregathor_b200.ops import gar as gar_ops
  base = torch.randn(9, 1030, device="cuda")
  G = base[:, 3:1004]   # not contiguous, not 16-byte aligned: crafted on a padded copy, written back
  before = base.clone()
  gamma, *_ = gar_ops.craft_byzantine_(G, [7, 8], "min-max", deviation="sign", return_details=True)
  expected = _ops.torch_optimized_row(before[:, 3:1004].cpu().contiguous(), [7, 8], "min-max", "sign", gamma)
  _equal_values(G[7], expected)
  _equal_values(G[8], expected)
  assert torch.equal(base[:7], before[:7]) and torch.equal(base[:, :3], before[:, :3]) and torch.equal(base[:, 1004:], before[:, 1004:])


def test_more_than_32_workers_use_the_torch_reference():
  from aggregathor_b200.ops import gar as gar_ops
  G = torch.randn(36, 999, generator=torch.Generator().manual_seed(8))
  Gd = G.cuda()
  gamma, A, B, C, T = gar_ops.craft_byzantine_(Gd, [33, 34, 35], "min-sum", deviation="std", return_details=True)
  expected = _ops.torch_craft_byzantine_(G.clone(), [33, 34, 35], "min-sum", None, deviation="std", return_details=True)
  assert len(A) == 33 and abs(gamma - expected[0]) <= 1e-6 * expected[0]
  _equal_values(Gd[35], _ops.torch_optimized_row(G, [33, 34, 35], "min-sum", "std", gamma))


def _manager(rule, n, k, mode, deviation, engine):
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate(rule, n, k, [])
  return Manager(experiment, gar, n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cuda", engine=engine, seed=7,
                 attack=attacks.instantiate(mode, n, k, ["deviation:" + deviation]), nb_real_byz=k)


@pytest.mark.parametrize("mode,deviation", [("min-max", "unit-vec"), ("min-sum", "std"), ("min-max", "sign")])
@pytest.mark.parametrize("rule,n", [("average", 11), ("median", 11), ("krum", 11), ("trimmed-mean", 11), ("mda", 11), ("bulyan", 11)])
def test_fused_engine_matches_the_baseline_engine(rule, n, mode, deviation):
  """Both engines run the crafting kernel at R = 1 on the same owned coordinates [0, d): same grid, same fold order, same bits."""
  fused = _manager(rule, n, 2, mode, deviation, "fused")
  base = _manager(rule, n, 2, mode, deviation, "baseline")
  assert fused.aggregation.name == "fused" and base.aggregation.name == "baseline"
  for _ in range(3):
    fused.train()
    base.train()
    torch.cuda.synchronize()
    assert fused.aggregation.last_craft == base.aggregation.last_craft
    assert fused.aggregation.last_craft[0] > 0
    for i in (n - 2, n - 1):
      assert torch.equal(_bits(fused.aggregation.visible_rows()[i]), _bits(base.aggregation.visible_rows()[i]))
  assert torch.equal(_bits(fused.params), _bits(base.params))
  fused.close()
  base.close()


def _gpus():
  return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_gpus() < 2, reason="needs at least 2 GPUs")
@pytest.mark.parametrize("mode", MODES)
def test_sharded_crafting_on_several_gpus(tmp_path, mode):
  """n = 8 over 2 or 4 ranks, both Byzantine workers on the last rank: every rank solves the same gamma from the exchanged sums, the
  crafted rows are the reference row for that gamma, and the baseline engine's gamma differs at most in its last bits."""
  nproc = 4 if _gpus() >= 4 else 2
  port = 29900 + os.getpid() % 90
  cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1", "--master-port", str(port),
         str(ROOT / "benchmarks" / "gar_bench.py"), "--gar-dim", "1000003", "--gar-iters", "3", "--gar-rules", "average,krum", "--gar-out", str(tmp_path),
         "--gar-attack", mode, "--gar-attack-args", "deviation:std", "--gar-dump-rows"]
  proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, cwd=str(ROOT), env=dict(os.environ, AGB_NVLS_REDUCE="1"))
  out = proc.stdout.decode(errors="replace")
  assert proc.returncode == 0, out[-4000:]
  results = json.loads((tmp_path / ("gar_bench_%d.json" % nproc)).read_text())["results"]
  for rule in ("average", "krum"):
    entry = results[rule]
    assert entry["attack"] == mode and entry["replicas_identical"], (rule, entry)
    gammas = entry["gamma_per_rank"]
    assert len(gammas) == nproc and len(set(gammas)) == 1 and gammas[0] > 0, (rule, entry)
    assert abs(gammas[0] - entry["baseline_gamma"]) <= 1e-5 * gammas[0], (rule, entry)
    dump = torch.load(tmp_path / ("gar_rows_%s_%d.pt" % (rule, nproc)))
    rows, byz = dump["rows"], dump["byzantine"]
    assert byz == [6, 7] and dump["gamma"] == gammas[0]
    expected = _ops.torch_optimized_row(rows, byz, mode, "std", dump["gamma"])   # from the honest rows, over all d coordinates
    for i in byz:
      _equal_values(rows[i], expected)
    # the engines differ only through gamma's last bits: |b - b'| <= |gamma - gamma'| * |p| + rounding of both rows
    assert entry["max_abs_diff_vs_baseline"] <= 1e-3, (rule, entry)

"""Omniscient attacks (ALIE, IPM) on sm_90a: the crafting kernel against the torch reference bit for bit, the fused engine against the
baseline engine through training, ALIE steering the Krum kernel, and the sharded crafting pass on several GPUs."""

import json
import os
import pathlib
import subprocess
import sys

import pytest
import torch

from aggregathor_b200 import aggregators, attacks, experiments
from aggregathor_b200.aggregators import FusedSpec, _ops
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
  """Seeded rows over four decades; with `honest` slots, NaN, +inf and -inf are sprinkled into three of them."""
  G = torch.randn(n, d, generator=torch.Generator().manual_seed(seed)) * torch.logspace(-2, 2, d)
  if honest is not None:
    G[honest[0], 3::101] = float("nan")
    G[honest[1 % len(honest)], 5::103] = float("inf")
    G[honest[-1], 7::107] = float("-inf")
  return G


def _cases():
  for n in (3, 8, 9, 17, 32):
    for k in sorted({1, max(1, n // 3), n - 2}):
      yield n, k


@pytest.mark.parametrize("d", [400003, 400000])
@pytest.mark.parametrize("n,k", list(_cases()))
def test_kernel_matches_the_reference_bit_for_bit(n, k, d):
  from aggregathor_b200.ops import gar as gar_ops
  for mode, non_finite in (("alie", False), ("ipm", False), ("alie", True), ("ipm", True)):
    byz = list(range(n - k, n)) if mode == "alie" else list(range(k))   # the Byzantine slots may come first too
    G = _matrix(n, d, seed=n * 31 + k + d, honest=[i for i in range(n) if i not in byz] if non_finite else None)
    coef = attacks.instantiate(mode, n, k, ["z:1.25"] if mode == "alie" else []).coef
    expected = _ops.torch_craft_byzantine_(G.clone(), byz, mode, coef)
    Gd = G.cuda()
    out = gar_ops.craft_byzantine_(Gd, byz, mode, coef)
    torch.cuda.synchronize()
    assert out is Gd
    for i in range(n):
      if i in byz:
        _equal_values(Gd[i], expected[i])
      else:
        assert torch.equal(_bits(Gd[i]), _bits(G[i])), i   # honest rows byte-identical
    if non_finite:
      assert bool(torch.isnan(Gd[byz[0]]).any())


def test_kernel_leaves_a_strided_caller_matrix_alone_outside_the_byzantine_rows():
  from aggregathor_b200.ops import gar as gar_ops
  base = torch.randn(9, 1030, device="cuda")
  G = base[:, 3:1004]   # not contiguous, not 16-byte aligned: crafted on a padded copy, written back
  before = base.clone()
  gar_ops.craft_byzantine_(G, [7, 8], "alie", 0.5)
  expected = _ops.torch_craft_byzantine_(before[:, 3:1004].cpu().contiguous(), [7, 8], "alie", 0.5)
  _equal_values(G[7:], expected[7:])
  assert torch.equal(base[:7], before[:7]) and torch.equal(base[:, :3], before[:, :3]) and torch.equal(base[:, 1004:], before[:, 1004:])


def test_more_than_32_workers_use_the_torch_reference():
  from aggregathor_b200.ops import gar as gar_ops
  G = torch.randn(36, 999)
  expected = _ops.torch_craft_byzantine_(G.clone(), [33, 34, 35], "ipm", 0.1)
  Gd = gar_ops.craft_byzantine_(G.cuda(), [33, 34, 35], "ipm", 0.1)
  assert torch.allclose(Gd.cpu(), expected, rtol=1e-6, atol=0)


def test_alie_steers_the_krum_kernel():
  """See `test_alie_steers_krum` of the CPU tests for why a Byzantine row wins at this size; ties go to the lower slot."""
  from aggregathor_b200.ops import gar as gar_ops
  n, k = 8, 2
  G = torch.randn(n, 10 ** 4, generator=torch.Generator().manual_seed(42)).cuda()
  gar_ops.craft_byzantine_(G, [6, 7], "alie", attacks.instantiate("alie", n, k, []).coef)
  out, _, info = gar_ops.aggregate(FusedSpec("krum", n, f=2, m=1), G, return_details=True)
  assert int(info[0].item()) == 1 and int(info[1].item()) == 1 << 6
  assert torch.equal(_bits(out), _bits(G[6]))


def _manager(rule, n, k, mode, engine):
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate(rule, n, k, [])
  return Manager(experiment, gar, n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cuda", engine=engine, seed=7,
                 attack=attacks.instantiate(mode, n, k, []), nb_real_byz=k)


@pytest.mark.parametrize("mode", ["alie", "ipm"])
@pytest.mark.parametrize("rule,n", [("average", 8), ("median", 8), ("krum", 8), ("trimmed-mean", 8), ("mda", 8), ("bulyan", 11)])
def test_fused_engine_matches_the_baseline_engine(rule, n, mode):
  fused = _manager(rule, n, 2, mode, "fused")
  base = _manager(rule, n, 2, mode, "baseline")
  assert fused.aggregation.name == "fused" and base.aggregation.name == "baseline"
  for _ in range(3):
    fused.train()
    base.train()
    torch.cuda.synchronize()
    assert torch.equal(_bits(fused.aggregation.visible_rows()[n - 1]), _bits(base.aggregation.visible_rows()[n - 1]))
  assert torch.equal(_bits(fused.params), _bits(base.params))
  fused.close()
  base.close()


def _gpus():
  return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_gpus() < 2, reason="needs at least 2 GPUs")
@pytest.mark.parametrize("mode", ["alie", "ipm"])
def test_sharded_crafting_on_several_gpus(tmp_path, mode):
  """n = 8 over 2 or 4 ranks: both Byzantine workers (slots 6, 7) live on the last rank, the other ranks host none and still craft
  their slices. `average` runs with the NVLS in-switch reduction, `krum` with the staging buffer."""
  nproc = 4 if _gpus() >= 4 else 2
  port = 29900 + os.getpid() % 90
  cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1", "--master-port", str(port),
         str(ROOT / "benchmarks" / "gar_bench.py"), "--gar-dim", "1000003", "--gar-iters", "3", "--gar-rules", "average,krum", "--gar-out", str(tmp_path),
         "--gar-attack", mode, "--gar-dump-rows"]
  proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, cwd=str(ROOT), env=dict(os.environ, AGB_NVLS_REDUCE="1"))
  out = proc.stdout.decode(errors="replace")
  assert proc.returncode == 0, out[-4000:]
  results = json.loads((tmp_path / ("gar_bench_%d.json" % nproc)).read_text())["results"]
  for rule in ("average", "krum"):
    entry = results[rule]
    assert entry["attack"] == mode and entry["replicas_identical"], (rule, entry)
    assert entry["max_abs_diff_vs_baseline"] == 0.0, (rule, entry)
    dump = torch.load(tmp_path / ("gar_rows_%s_%d.pt" % (rule, nproc)))
    rows, byz = dump["rows"], dump["byzantine"]
    assert byz == [6, 7] and 8 // nproc >= 2   # both on the last rank
    expected = _ops.torch_byzantine_row(rows, byz, mode, dump["coef"])   # from the honest rows, over all d coordinates
    for i in byz:
      _equal_values(rows[i], expected)

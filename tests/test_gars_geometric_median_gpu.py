"""sm_90a geometric median: the kernel's output replayed bit for bit from the host median and the kernel's own distances, the
distances against float64, the fused engine with every optimizer, training under ALIE (fused vs baseline), the fall-backs, the
parameter checks and the multi-GPU engine."""

import json
import os
import pathlib
import subprocess
import sys

import numpy as np
import pytest
import torch

from aggregathor_b200 import aggregators, attacks, experiments
from aggregathor_b200.aggregators import FusedSpec, _ops
from aggregathor_b200.engine.flat import FlatLayout
from aggregathor_b200.engine.optimizers import optimizers
from aggregathor_b200.engine.schedules import build
from aggregathor_b200.engine.trainer import Manager

pytestmark = pytest.mark.gpu
ROOT = pathlib.Path(__file__).resolve().parent.parent


def _data(n, d, seed, outliers=0, non_finite=False):
  gen = torch.Generator().manual_seed(seed)
  G = torch.randn(n, d, generator=gen)
  for k in range(outliers):
    G[n - 1 - k] = G[n - 1 - k] * 30 + 5
  if non_finite:   # rows 0 and 1 at disjoint coordinates: every median stays finite, both rows are excluded
    G[0, 3::11] = float("nan")
    G[1, 5::11] = float("inf")
    G[1, 7::11] = float("-inf")
  return G


def _equal_bits(a, b):
  a, b = a.cpu(), b.cpu()
  assert a.dtype == b.dtype and a.shape == b.shape
  nan = torch.isnan(a)
  assert torch.equal(nan, torch.isnan(b))
  diff = (a[~nan].view(torch.int32) != b[~nan].view(torch.int32)).nonzero()
  assert diff.numel() == 0, (int(diff[0]), float(a[~nan][diff[0]]), float(b[~nan][diff[0]]))


def _replay(X, z0, dists, nu):
  """Step 2 of the definition in NumPy fp32 (correctly rounded sqrt and division, no FMA) with the given distances [T, n]; returns
  z_T and the iterates z_0 .. z_{T-1} the distances belong to."""
  one, nu = np.float32(1), np.float32(nu)
  z, iterates = z0, []
  for D in dists:
    iterates.append(z)
    kept = [i for i in range(X.shape[0]) if np.isfinite(D[i])]
    if not kept:
      continue
    S, num = np.float32(0), np.zeros_like(z)
    for i in kept:
      beta = one / np.maximum(nu, np.sqrt(D[i]))
      S = np.float32(S + beta)
      num = num + beta * X[i]
    z = num / S
  return z, iterates


@pytest.mark.parametrize("iterations", [1, 3, 16])
@pytest.mark.parametrize("d", [4096, 1003])
@pytest.mark.parametrize("n", [3, 5, 8, 9, 16, 17, 32])
def test_kernel_replays_bit_for_bit(n, d, iterations):
  from aggregathor_b200.ops import gar as gar_ops
  nu = 1e-6
  G = _data(n, d, seed=n * 31 + d + iterations, outliers=max(1, (n - 1) // 4), non_finite=n >= 5)
  spec = FusedSpec("geometric-median", n, f=(n - 1) // 2, iterations=iterations, nu=nu)
  out, dist, _ = gar_ops.aggregate(spec, G.cuda(), return_details=True)
  dist = dist.cpu().numpy()
  assert dist.shape == (iterations, n)
  X = G.numpy()
  z0 = _ops.host_median(G).numpy()
  z, iterates = _replay(X, z0, dist, spec.nu)
  _equal_bits(out, torch.from_numpy(z))
  assert bool(torch.isfinite(out).all())
  for t, zt in enumerate(iterates):
    exact = ((X.astype(np.float64) - zt.astype(np.float64)) ** 2).sum(axis=1)
    finite = np.isfinite(exact)
    assert np.array_equal(finite, np.isfinite(dist[t])), t
    bound = (d + 2) * 2.0 ** -24 * exact[finite]
    assert (np.abs(dist[t][finite].astype(np.float64) - exact[finite]) <= bound).all(), t
  if n >= 5:
    assert not np.isfinite(dist[:, :2]).any() and np.isfinite(dist[:, 2:]).all()


def test_no_kept_row_returns_the_median():
  from aggregathor_b200.ops import gar as gar_ops
  G = _data(9, 2001, seed=3)
  G[:, 17] = float("nan")   # the median is NaN there, so is every distance
  out, dist, _ = gar_ops.aggregate(FusedSpec("geometric-median", 9, iterations=4), G.cuda(), return_details=True)
  _equal_bits(out, _ops.host_median(G))
  assert not np.isfinite(dist.cpu().numpy()).any()


@pytest.mark.parametrize("opt", ["sgd", "adam", "rmsprop", "adagrad", "adadelta"])
def test_fused_optimizers_single_rank(opt):
  """The fused kernel (R = 1) aggregates exactly like the stand-alone op; its parameters stay close to HostAggregation's (the host
  library adds the distances in another order)."""
  from aggregathor_b200.ops import gar as gar_ops
  from aggregathor_b200.parallel.aggregation import FusedAggregation, HostAggregation
  layout = FlatLayout()
  layout.add("w", (1000, 37))
  layout.add("b", (37,))
  layout.freeze()
  gar = aggregators.instantiate("geometric-median", 8, 2, ["iterations:3"])
  fused = FusedAggregation(gar, layout, 8, build(optimizers, "optimizer", opt, []), device="cuda", keep_aggregate=True)
  host = HostAggregation(gar, layout, 8, build(optimizers, "optimizer", opt, []), device="cpu")
  assert not fused.overlappable and fused.staging is None
  gen = torch.Generator().manual_seed(5)
  init = torch.randn(layout.padded_size, generator=gen)
  fused.params.copy_(init)
  host.params.copy_(init)
  for step in range(3):
    G = torch.randn(8, layout.padded_size, generator=gen) * 0.1
    G[7] += 3.0
    G[6, ::5] -= 2.0
    fused.grads.copy_(G)
    host.grads.copy_(G)
    fused.step(0.05)
    host.step(0.05)
    torch.cuda.synchronize()
    _equal_bits(fused.last_aggregate, gar_ops.aggregate(gar.fused_spec(), G.cuda()))
    assert float((fused.last_aggregate.cpu() - host.last_aggregate).abs().max()) <= 1e-5
    assert float((fused.params.cpu() - host.params).abs().max()) <= 1e-4 * max(1.0, float(host.params.abs().max()))


def _manager(n, k, engine):
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate("geometric-median", n, k, [])
  return Manager(experiment, gar, n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cuda", engine=engine, seed=7,
                 attack=attacks.instantiate("alie", n, k, []), nb_real_byz=k)


def test_fused_engine_matches_the_baseline_engine_under_alie():
  fused = _manager(8, 2, "fused")
  base = _manager(8, 2, "baseline")
  assert fused.aggregation.name == "fused" and base.aggregation.name == "baseline"
  for _ in range(3):
    fused.train()
    base.train()
    torch.cuda.synchronize()
  assert torch.equal(fused.params.cpu().view(torch.int32), base.params.cpu().view(torch.int32))
  fused.close()
  base.close()


def test_double_inputs_stay_double_and_more_than_32_workers_fall_back():
  from aggregathor_b200.ops import gar as gar_ops
  G = _data(9, 3001, seed=4, outliers=2).double()
  out = gar_ops.aggregate(FusedSpec("geometric-median", 9, f=2), G.cuda())
  assert out.dtype == torch.float64
  ref = _ops.host_geometric_median(G, 3, 1e-6)
  assert float((out.cpu() - ref).abs().max()) <= 1e-12 * max(1.0, float(ref.abs().max()))
  G = _data(36, 2001, seed=6, outliers=3)
  out = gar_ops.aggregate(FusedSpec("geometric-median", 36, f=3), G.cuda())
  assert float((out.cpu().double() - _ops.host_geometric_median(G.double(), 3, 1e-6)).abs().max()) < 1e-5
  gar = aggregators.instantiate("geometric-median", 8, 2, [])
  G = _data(8, 3000, seed=11, outliers=2)
  _equal_bits(gar.aggregate(list(G.cuda())), gar_ops.aggregate(gar.fused_spec(), G.cuda()))


def test_kernel_rejects_invalid_parameters():
  from aggregathor_b200.ops import gar as gar_ops
  G = torch.randn(8, 64, device="cuda")
  for kwargs in ({"f": 4}, {"iterations": 0}, {"iterations": 17}, {"nu": 0.0}, {"nu": -1.0}, {"nu": float("inf")}, {"nu": float("nan")}):
    with pytest.raises(RuntimeError, match="status 115"):
      gar_ops.aggregate(FusedSpec("geometric-median", 8, **kwargs), G)


def _gpus():
  return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_gpus() < 2, reason="needs at least 2 GPUs")
def test_fused_matches_baseline_on_all_ranks(tmp_path):
  nproc = max(r for r in range(1, min(_gpus(), 8) + 1) if 8 % r == 0)
  port = 29900 + os.getpid() % 90
  cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1", "--master-port", str(port),
         str(ROOT / "benchmarks" / "gar_bench.py"), "--gar-dim", "1000003", "--gar-iters", "3", "--gar-rules", "geometric-median", "--gar-out", str(tmp_path)]
  proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, cwd=str(ROOT))
  out = proc.stdout.decode(errors="replace")
  assert proc.returncode == 0, out[-4000:]
  results = json.loads((tmp_path / ("gar_bench_%d.json" % nproc)).read_text())["results"]
  entry = results["geometric-median"]
  assert entry["replicas_identical"], entry
  assert entry["max_abs_diff_vs_baseline"] < 1e-4, entry

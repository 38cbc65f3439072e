"""sm_90a centered clipping: three calls in a row with the center carried over, replayed bit for bit from the kernel's own distances,
the distances against float64, fused vs baseline training with worker momentum under ALIE and flip, the fall-backs, the parameter
checks and the multi-GPU engine."""

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
from aggregathor_b200.engine.trainer import Manager

pytestmark = pytest.mark.gpu
ROOT = pathlib.Path(__file__).resolve().parent.parent


def _data(n, d, seed, outliers=0, non_finite=False):
  gen = torch.Generator().manual_seed(seed)
  G = torch.randn(n, d, generator=gen)
  for k in range(outliers):
    G[n - 1 - k] = G[n - 1 - k] * 30 + 5
  if non_finite:   # rows 0 and 1 have non-finite distances at every iteration: both are skipped
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


def _replay(X, z0, dists, tau):
  """The definition in NumPy fp32 (correctly rounded sqrt and division, no FMA) with the given distances [T, n]; returns z_T and the
  iterates z_0 .. z_{T-1} the distances belong to."""
  one, tau, count = np.float32(1), np.float32(tau), np.float32(X.shape[0])
  z, iterates = z0, []
  for D in dists:
    iterates.append(z)
    kept = [i for i in range(X.shape[0]) if np.isfinite(D[i])]
    if not kept:
      continue
    u = np.zeros_like(z)
    for i in kept:
      s = np.sqrt(np.float32(D[i]))
      c = one if s <= tau else np.float32(tau / s)
      u = u + c * (X[i] - z)
    z = z + u / count
  return z, iterates


@pytest.mark.parametrize("iterations", [1, 3, 16])
@pytest.mark.parametrize("n", [3, 8, 9, 17, 32])
def test_kernel_replays_bit_for_bit_over_three_calls(n, iterations):
  from aggregathor_b200.ops import gar as gar_ops
  d, tau = 2003, 2.0
  spec = FusedSpec("centered-clipping", n, f=(n - 1) // 2, iterations=iterations, tau=tau)
  center = torch.zeros(d, device="cuda")
  z = np.zeros(d, dtype=np.float32)
  for call in range(3):
    G = _data(n, d, seed=n * 31 + iterations * 7 + call, outliers=max(1, (n - 1) // 4), non_finite=n >= 8)
    out, dist, _ = gar_ops.aggregate(spec, G.cuda(), return_details=True, center=center)
    dist = dist.cpu().numpy()
    assert dist.shape == (iterations, n)
    X = G.numpy()
    z, iterates = _replay(X, z, dist, spec.tau)
    _equal_bits(out, torch.from_numpy(z))
    _equal_bits(center, torch.from_numpy(z))
    assert bool(torch.isfinite(out).all())
    for t, zt in enumerate(iterates):
      exact = ((X.astype(np.float64) - zt.astype(np.float64)) ** 2).sum(axis=1)
      finite = np.isfinite(exact)
      assert np.array_equal(finite, np.isfinite(dist[t])), t
      bound = (d + 2) * 2.0 ** -24 * exact[finite]
      assert (np.abs(dist[t][finite].astype(np.float64) - exact[finite]) <= bound).all(), t
    if n >= 8:
      assert not np.isfinite(dist[:, :2]).any() and np.isfinite(dist[:, 2:]).all()


def test_kernel_matches_the_host_library_on_aligned_rows():
  """d a multiple of 4 (the center is updated in place, no padded copy); the host library adds the distances in another order."""
  from aggregathor_b200.ops import gar as gar_ops
  n, d = 9, 40000
  spec = FusedSpec("centered-clipping", n, f=2, iterations=3, tau=5.0)
  center, host_center = torch.zeros(d, device="cuda"), torch.zeros(d)
  for call in range(3):
    G = _data(n, d, seed=call, outliers=2)
    out = gar_ops.aggregate(spec, G.cuda(), center=center)
    ref = _ops.host_centered_clipping(G, 3, 5.0, host_center)
    assert float((out.cpu() - ref).abs().max()) <= 1e-5
  assert float((center.cpu() - host_center).abs().max()) <= 1e-5


def _manager(engine, attack, k=2, n=8):
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate("centered-clipping", n, k, ["iterations:3", "tau:1"])
  return Manager(experiment, gar, n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cuda", engine=engine, seed=7,
                 attack=attacks.instantiate(attack, n, k, []), nb_real_byz=k, worker_momentum=0.9, worker_momentum_dampening=0.1)


@pytest.mark.parametrize("attack", ["alie", "flip"])
def test_fused_engine_matches_the_baseline_engine(attack):
  fused = _manager("fused", attack)
  base = _manager("baseline", attack)
  assert fused.aggregation.name == "fused" and base.aggregation.name == "baseline"
  for _ in range(3):
    fused.train()
    base.train()
    torch.cuda.synchronize()
  _equal_bits(fused.params, base.params)
  _equal_bits(fused.aggregation.center, base.aggregation.center)
  _equal_bits(fused.worker_momentum, base.worker_momentum)
  assert bool(fused.aggregation.center.any())
  fused.close()
  base.close()


def test_double_inputs_and_more_than_32_workers_fall_back():
  from aggregathor_b200.ops import gar as gar_ops
  G = _data(9, 3001, seed=4, outliers=2).double()
  center = torch.zeros(3001, dtype=torch.float64, device="cuda")
  out = gar_ops.aggregate(FusedSpec("centered-clipping", 9, f=2, iterations=2, tau=3.0), G.cuda(), center=center)
  assert out.dtype == torch.float64 and torch.equal(out, center)
  host_center = torch.zeros(3001, dtype=torch.float64)
  ref = _ops.host_centered_clipping(G, 2, 3.0, host_center)
  assert float((out.cpu() - ref).abs().max()) <= 1e-12 * max(1.0, float(ref.abs().max()))
  G = _data(36, 2001, seed=6, outliers=3)
  center = torch.zeros(2001, device="cuda")
  out = gar_ops.aggregate(FusedSpec("centered-clipping", 36, f=3, iterations=2, tau=3.0), G.cuda(), center=center)
  ref = _ops.host_centered_clipping(G.double(), 2, 3.0, torch.zeros(2001, dtype=torch.float64))
  assert float((out.cpu().double() - ref).abs().max()) < 1e-5
  gar = aggregators.instantiate("centered-clipping", 8, 2, [])
  G = _data(8, 3000, seed=11, outliers=2)
  mine = torch.zeros(3000, device="cuda")
  _equal_bits(gar.aggregate(list(G.cuda())), gar_ops.aggregate(gar.fused_spec(), G.cuda(), center=mine))


def test_kernel_rejects_invalid_parameters():
  from aggregathor_b200.ops import gar as gar_ops
  G = torch.randn(8, 64, device="cuda")
  center = torch.zeros(64, device="cuda")
  for kwargs in ({"f": 4}, {"iterations": 0}, {"iterations": 17}, {"tau": 0.0}, {"tau": -1.0}, {"tau": float("inf")}, {"tau": float("nan")}):
    with pytest.raises(RuntimeError, match="status 116"):
      gar_ops.aggregate(FusedSpec("centered-clipping", 8, **kwargs), G, center=center)
  launcher = gar_ops.FusedLauncher(G.device, 8)
  out = torch.empty(64, device="cuda")
  with pytest.raises(RuntimeError, match="status 116"):   # no center buffer
    launcher.launch(FusedSpec("centered-clipping", 8), [G.data_ptr() + i * 64 * 4 for i in range(8)], 0, 64, agg_out=out)


def _gpus():
  return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_gpus() < 2, reason="needs at least 2 GPUs")
def test_fused_matches_baseline_on_all_ranks(tmp_path):
  nproc = max(r for r in range(1, min(_gpus(), 8) + 1) if 8 % r == 0)
  port = 29800 + os.getpid() % 90
  cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1", "--master-port", str(port),
         str(ROOT / "benchmarks" / "gar_bench.py"), "--gar-dim", "1000003", "--gar-iters", "3", "--gar-rules", "centered-clipping",
         "--gar-rule-args", "iterations:3", "tau:1", "--gar-out", str(tmp_path)]
  proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, cwd=str(ROOT))
  out = proc.stdout.decode(errors="replace")
  assert proc.returncode == 0, out[-4000:]
  results = json.loads((tmp_path / ("gar_bench_%d.json" % nproc)).read_text())["results"]
  entry = results["centered-clipping"]
  assert entry["replicas_identical"], entry
  assert entry["max_abs_diff_vs_baseline"] < 1e-4, entry

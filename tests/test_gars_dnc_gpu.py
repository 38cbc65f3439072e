"""sm_90a DnC: the kernel replayed bit for bit from its own sampled distances (with and without NNM), the distances against float64
on the sampler's coordinates, fused vs baseline training under CUDA-graph replay, the fall-backs, the parameter checks and the
multi-GPU engine."""

import json
import os
import pathlib
import subprocess
import sys

import numpy as np
import pytest
import torch

from aggregathor_b200 import aggregators
from aggregathor_b200.aggregators import FusedSpec, _ops
from aggregathor_b200.engine.flat import FlatLayout
from aggregathor_b200.engine.optimizers import optimizers
from aggregathor_b200.engine.schedules import build
from aggregathor_b200.parallel.aggregation import BaselineAggregation, FusedAggregation

pytestmark = pytest.mark.gpu
ROOT = pathlib.Path(__file__).resolve().parent.parent


def _data(n, d, seed, outliers=0, non_finite=False):
  gen = torch.Generator().manual_seed(seed)
  G = torch.randn(n, d, generator=gen)
  for k in range(outliers):
    G[n - 1 - k] = G[n - 1 - k] * 30 + 5
  if non_finite:
    G[0, 3::11] = float("nan")
    G[1, 5::11] = float("inf")
  return G


def _equal_bits(a, b):
  a, b = a.cpu(), b.cpu()
  assert a.dtype == b.dtype and a.shape == b.shape
  nan = torch.isnan(a)
  assert torch.equal(nan, torch.isnan(b))
  diff = (a[~nan].view(torch.int32) != b[~nan].view(torch.int32)).nonzero()
  assert diff.numel() == 0, (int(diff[0]), float(a[~nan][diff[0]]), float(b[~nan][diff[0]]))


def _mask_bits(mask):
  return sum(1 << i for i in range(len(mask)) if mask[i])


def _replay(spec, X, out, dist, info, step):
  """Check the kernel's [T, n, n] distances against float64 on the sampler's coordinates, its masks against `dnc_select` on those
  distances, and its output against the NumPy mean of the selected rows."""
  n, d = X.shape
  T = spec.iterations
  dist = dist.cpu().numpy()
  assert dist.shape == (T, n, n)
  for t in range(T):
    S = X[:, _ops.dnc_sample(d, spec.subsample, spec.seed, step, t)].astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
      exact = ((S[:, None, :] - S[None, :, :]) ** 2).sum(axis=2)
    np.fill_diagonal(exact, 0.0)   # a row with a NaN is at distance 0 from itself
    finite = np.isfinite(exact)
    assert np.array_equal(finite, np.isfinite(dist[t])), t
    bound = (S.shape[1] + 2) * 2.0 ** -24 * exact[finite]
    assert (np.abs(dist[t][finite].astype(np.float64) - exact[finite]) <= bound).all(), t
  masks, good = _ops.dnc_select(dist, spec.removed)
  info = info.cpu().tolist()
  assert info[0] == 1 and info[1] & 0xffffffff == _mask_bits(good)
  assert [v & 0xffffffff for v in info[96:96 + T]] == [_mask_bits(m) for m in masks]
  acc = np.zeros(d, dtype=np.float32)
  for i in range(n):
    if good[i]:
      acc = acc + X[i]
  _equal_bits(out, torch.from_numpy(acc / np.float32(good.sum())))
  return good


@pytest.mark.parametrize("T", [1, 3])
@pytest.mark.parametrize("n", [3, 8, 9, 17, 32])
def test_kernel_replays_bit_for_bit(n, T):
  from aggregathor_b200.ops import gar as gar_ops
  d, f = 20003, (n - 1) // 2
  c = 1.0 if n - T * f >= 1 else 1.0 / T
  spec = FusedSpec("dnc", n, f=f, iterations=T, subsample=3000, c=c, seed=5)
  for step in (1, 2):
    G = _data(n, d, seed=n * 7 + T + step, outliers=max(1, f // 2), non_finite=n >= 8)
    out, dist, info = gar_ops.aggregate(spec, G.cuda(), return_details=True, step=step)
    good = _replay(spec, G.numpy(), out, dist, info, step)
    if n >= 8 and spec.removed >= 2:   # every iteration can remove both non-finite rows
      assert not good[0] and not good[1] and bool(torch.isfinite(out).all())


@pytest.mark.parametrize("n", [8, 17])
def test_kernel_replays_bit_for_bit_after_nnm(n):
  from aggregathor_b200.ops import gar as gar_ops
  d, f = 10001, 2
  spec = FusedSpec("dnc", n, f=f, iterations=2, subsample=2000, seed=1, mix="nnm")
  G = _data(n, d, seed=n, outliers=f)
  out, dist, info, (raw, nnm_masks) = gar_ops.aggregate(spec, G.cuda(), return_details=True, step=3)
  member = _ops.nnm_select(raw.cpu(), f)
  assert torch.equal(nnm_masks.cpu(), _ops.nnm_bits(member))
  mixed = _ops.torch_nnm_mix(G, member, f)
  _replay(spec, mixed.numpy(), out, dist, info, 3)


def test_full_sample_and_tiny_domains():
  from aggregathor_b200.ops import gar as gar_ops
  for n, d, b in ((5, 3, 10), (4, 1, 1), (6, 777, 777), (6, 777, 100000)):
    spec = FusedSpec("dnc", n, f=1, iterations=2, subsample=b)
    G = _data(n, d, seed=d)
    out, dist, info = gar_ops.aggregate(spec, G.cuda(), return_details=True, step=4)
    _replay(spec, G.numpy(), out, dist, info, 4)


def _engines(n=8, f=2, d=50003, device_state=False):
  layout = FlatLayout()
  layout.add("w", (d,))
  layout.freeze()
  gar = aggregators.instantiate("dnc", n, f, ["iterations:2", "subsample:4000", "seed:7"])
  fused = FusedAggregation(gar, layout, n, build(optimizers, "optimizer", "sgd", []), device="cuda", keep_aggregate=True, device_state=device_state)
  base = BaselineAggregation(gar, layout, n, build(optimizers, "optimizer", "sgd", []), device="cuda")
  init = torch.randn(layout.padded_size, generator=torch.Generator().manual_seed(1)).cuda()
  fused.params.copy_(init)
  base.params.copy_(init)
  return fused, base, layout.padded_size


def test_fused_engine_matches_the_baseline_engine_under_graph_replay():
  n, f = 8, 2
  fused, base, d = _engines(n, f, device_state=True)
  grads = [_data(n, d, seed=10 + k, outliers=f).cuda() for k in range(4)]
  # step 1 eagerly (allocations), then capture one step and replay it
  fused.grads.copy_(grads[0])
  fused.step(0.1)
  base.grads.copy_(grads[0])
  base.step(0.1)
  torch.cuda.synchronize()
  _equal_bits(fused.params, base.params)
  graph = torch.cuda.CUDAGraph()
  stream = torch.cuda.Stream()
  fused.prepare(0.1)
  fused.grads.copy_(grads[1])
  torch.cuda.synchronize()
  with torch.cuda.graph(graph, stream=stream):
    fused.step(prepared=True)
  graph.replay()
  base.grads.copy_(grads[1])
  base.step(0.1)
  torch.cuda.synchronize()
  samples = []
  for k in (2, 3):   # the same rows twice: only the step key can change the distances
    fused.prepare(0.1)
    fused.grads.copy_(grads[2])
    graph.replay()
    base.grads.copy_(grads[2])
    base.step(0.1)
    torch.cuda.synchronize()
    _equal_bits(fused.params, base.params)
    _equal_bits(fused.launcher.dnc_dist_out[:2 * n * n], base_launcher_dists(base, n)[:2 * n * n])   # T = 2 iterations
    samples.append(fused.launcher.dnc_dist_out[:2 * n * n].clone())
  assert int(fused.step_dev.item()) == fused.updates == base.updates == 4
  assert not torch.equal(samples[0], samples[1])
  X = grads[2].cpu().numpy().astype(np.float64)   # and they are the distances of the samples of step 4
  S = X[:, _ops.dnc_sample(d, 4000, 7, 4, 0)]
  exact = ((S[:, None, :] - S[None, :, :]) ** 2).sum(axis=2)
  assert np.allclose(samples[1][:n * n].view(n, n).cpu().numpy(), exact, rtol=1e-4)


def base_launcher_dists(base, n):
  from aggregathor_b200.ops import gar as gar_ops
  return gar_ops._launcher(base._gathered.device, n).dnc_dist_out


def test_double_inputs_and_more_than_32_workers_fall_back():
  from aggregathor_b200.ops import gar as gar_ops
  G = _data(9, 3001, seed=4, outliers=2).double()
  spec = FusedSpec("dnc", 9, f=2, iterations=2, subsample=500)
  out = gar_ops.aggregate(spec, G.cuda(), step=3)
  assert out.dtype == torch.float64
  assert torch.equal(out.cpu(), _ops.torch_dnc(G, 2, 2, 500, 1.0, 0, 3))
  G = _data(40, 2001, seed=6, outliers=3)
  out = gar_ops.aggregate(FusedSpec("dnc", 40, f=3, iterations=1, subsample=700), G.cuda(), step=2)
  ref = _ops.torch_dnc(G.cuda(), 3, 1, 700, 1.0, 0, 2)
  _equal_bits(out, ref)
  gar = aggregators.instantiate("dnc", 8, 2, [])
  G = _data(8, 3000, seed=11, outliers=2).cuda()
  _equal_bits(gar.aggregate(list(G)), gar_ops.aggregate(gar.fused_spec(), G, step=1))


def test_kernel_rejects_invalid_parameters():
  from aggregathor_b200.ops import gar as gar_ops
  G = torch.randn(8, 64, device="cuda")
  for kwargs in ({"f": 4}, {"iterations": 0}, {"iterations": 9}, {"subsample": 0}, {"subsample": (1 << 20) + 1}, {"f": 3, "iterations": 3},
                 {"f": -1}):
    with pytest.raises(RuntimeError, match="status 119"):
      gar_ops.aggregate(FusedSpec("dnc", 8, **kwargs), G, step=1)
  launcher = gar_ops.FusedLauncher(G.device, 8)
  out = torch.empty(64, device="cuda")
  with pytest.raises(RuntimeError, match="status 119"):   # a negative step key reaching the kernel (ops.gar.aggregate refuses it first)
    launcher.launch(FusedSpec("dnc", 8, f=2), [G.data_ptr() + i * 64 * 4 for i in range(8)], 0, 64, agg_out=out, step=-1)
  with pytest.raises(Exception, match="step key"):
    gar_ops.aggregate(FusedSpec("dnc", 8, f=2), G, step=-1)


def test_gar_bench_runs_dnc(tmp_path):
  cmd = [sys.executable, str(ROOT / "benchmarks" / "gar_bench.py"), "--gar-dim", "200003", "--gar-iters", "3", "--gar-rules", "krum,dnc",
         "--gar-rule-args", "iterations:2", "subsample:5000", "--gar-out", str(tmp_path)]
  proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, cwd=str(ROOT))
  out = proc.stdout.decode(errors="replace")
  assert proc.returncode == 0, out[-4000:]
  entry = json.loads((tmp_path / "gar_bench_1.json").read_text())["results"]["dnc"]
  assert entry["replicas_identical"] and entry["max_abs_diff_vs_baseline"] == 0.0 and entry["masks_agree"], entry


def _gpus():
  return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_gpus() < 2, reason="needs at least 2 GPUs")
def test_fused_matches_baseline_on_all_ranks(tmp_path):
  nproc = max(r for r in range(1, min(_gpus(), 8) + 1) if 8 % r == 0)
  port = 29800 + os.getpid() % 90
  cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1", "--master-port", str(port),
         str(ROOT / "benchmarks" / "gar_bench.py"), "--gar-dim", "1000003", "--gar-iters", "3", "--gar-rules", "dnc",
         "--gar-rule-args", "iterations:2", "--gar-out", str(tmp_path)]
  proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, cwd=str(ROOT))
  out = proc.stdout.decode(errors="replace")
  assert proc.returncode == 0, out[-4000:]
  entry = json.loads((tmp_path / ("gar_bench_%d.json" % nproc)).read_text())["results"]["dnc"]
  assert entry["replicas_identical"] and entry["masks_agree"], entry
  assert entry["max_abs_diff_vs_baseline"] < 1e-4, entry

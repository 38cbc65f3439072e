"""sm_90a adaptive robust clipping (ARC) inside the aggregation kernel: every rule replayed bit for bit on NumPy-clipped (and, with
"arc+nnm", NumPy-mixed) rows from the kernel's own norms, factors and masks, the norms against float64, the fall-backs, the status
codes, fused vs baseline training with worker momentum under ALIE and flip, and the multi-GPU engine."""

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
RULES = ["average", "average-nan", "median", "averaged-median", "krum", "bulyan", "trimmed-mean", "mda", "geometric-median",
         "centered-clipping", "dnc"]


def _data(n, d, seed, outliers=0, non_finite=False):
  gen = torch.Generator().manual_seed(seed)
  G = torch.randn(n, d, generator=gen)
  for k in range(outliers):
    G[n - 1 - k] = G[n - 1 - k] * 30 + 5
  if non_finite:   # row 0 has NaNs (a NaN norm), row 1 a few infinities (an infinite norm): both are clipped first
    G[0, 3::11] = float("nan")
    G[1, 5::97] = float("inf")
  return G


def _equal_bits(a, b):
  a, b = torch.as_tensor(a).cpu(), torch.as_tensor(b).cpu()
  assert a.dtype == b.dtype and a.shape == b.shape
  nan = torch.isnan(a)
  assert torch.equal(nan, torch.isnan(b))
  diff = (a[~nan].view(torch.int32) != b[~nan].view(torch.int32)).nonzero()
  assert diff.numel() == 0, (int(diff[0]), float(a[~nan][diff[0]]), float(b[~nan][diff[0]]))


def _np_clip(X, c):
  """y_i = x_i * c_i in NumPy fp32, for the rows whose factor is not 1."""
  Y = X.copy()
  with np.errstate(over="ignore", invalid="ignore"):
    for i in range(X.shape[0]):
      if not c[i] == 1.0:
        Y[i] = X[i] * np.float32(c[i])
  return Y


def _np_mix(X, masks, f):
  """NNM in NumPy fp32: members of N_i (bit masks) added in ascending order from +0, one division."""
  n = X.shape[0]
  Y = np.empty_like(X)
  with np.errstate(over="ignore", invalid="ignore"):
    for i in range(n):
      s = np.zeros(X.shape[1], dtype=np.float32)
      for j in range(n):
        if (int(masks[i]) >> j) & 1:
          s = s + X[j]
      Y[i] = s / np.float32(n - f)
  return Y


def _spec(rule, n, mix):
  f = {3: 1, 8: 2, 9: 2, 17: 4, 32: 7}[n]
  if rule == "bulyan":
    f = (n - 3) // 4
  if rule == "mda":
    f = min(f, 5)
  kwargs = {"geometric-median": dict(iterations=3), "centered-clipping": dict(iterations=3, tau=2.0),
            "dnc": dict(iterations=2, subsample=700, seed=5)}.get(rule, {})
  m = n - f - 2 if rule in ("krum", "bulyan") else 0
  beta = n - 4 * f - 2 if rule == "bulyan" else (n - f if rule == "averaged-median" else 0)
  return FusedSpec(rule, n, f=f, m=m, beta=beta, mix=mix, **kwargs), f


def _within_bound(dist, X64):
  """NNM's distances, off-diagonal pairs, within the fp32 bound of float64."""
  with np.errstate(invalid="ignore", over="ignore"):
    exact = ((X64[:, None, :] - X64[None, :, :]) ** 2).sum(axis=2)
  off = ~np.eye(X64.shape[0], dtype=bool)
  exact, dist = exact[off], dist[off]
  finite = np.isfinite(exact)
  assert np.array_equal(finite, np.isfinite(dist))
  bound = (X64.shape[1] + 2) * 2.0 ** -24 * exact[finite]
  assert (np.abs(dist[finite].astype(np.float64) - exact[finite]) <= bound).all()


def _norms_within_bound(N, X64):
  with np.errstate(invalid="ignore", over="ignore"):
    exact = (X64 ** 2).sum(axis=1)
  assert np.array_equal(np.isnan(exact), np.isnan(N)) and np.array_equal(np.isinf(exact), np.isinf(N))
  finite = np.isfinite(exact)
  bound = (X64.shape[1] + 2) * 2.0 ** -24 * exact[finite]
  assert (np.abs(N[finite].astype(np.float64) - exact[finite]) <= bound).all()


@pytest.mark.parametrize("mix", ["arc", "arc+nnm"])
@pytest.mark.parametrize("n", [3, 8, 9, 17, 32])
@pytest.mark.parametrize("rule", RULES)
def test_kernel_replays_bit_for_bit(rule, n, mix):
  from aggregathor_b200.ops import gar as gar_ops
  if rule == "krum" and n == 3:
    pytest.skip("Krum needs n - f - 2 >= 1")
  if rule == "bulyan" and n < 7:
    pytest.skip("Bulyan needs n >= 4 f + 3 with f >= 1")
  spec, f = _spec(rule, n, mix)
  plain = spec.with_mix(None)
  k = _ops.arc_clip_count(n, f)
  d = 2003
  calls = 3 if rule in ("centered-clipping", "dnc") else 1
  center, center_plain = torch.zeros(d, device="cuda"), torch.zeros(d, device="cuda")
  for call in range(calls):
    G = _data(n, d, seed=n * 17 + len(rule) + call + len(mix), outliers=max(1, f // 2), non_finite=n >= 8)
    state = {"center": center} if rule == "centered-clipping" else {"step": 11 + 7 * call} if rule == "dnc" else {}
    out, dist, info, *details = gar_ops.aggregate(spec, G.cuda(), return_details=True, **state)
    N, c = (t.cpu() for t in details[-1])
    X = G.numpy()
    # the kernel's norms are within the fp32 bound of float64, its factors are the selection on those very norms
    _norms_within_bound(N.numpy(), X.astype(np.float64))
    factors, clipped = _ops.arc_factors(N, f)
    _equal_bits(c, factors)
    # two non-finite norms (n >= 8): the threshold is finite when k >= 2; with k = 1 it is the NaN row and nothing is clipped
    assert int(clipped.sum()) == (k if n < 8 or k >= 2 else 0)
    Y = _np_clip(X, c.numpy())
    if n >= 8 and k >= 2:   # the NaN row and the infinite row are clipped: NaN, and 0 (NaN where it was infinite)
      assert bool(clipped[0]) and bool(clipped[1]) and np.isnan(Y[0]).all() and np.nanmax(np.abs(Y[1])) == 0.0
    if mix == "arc+nnm":
      raw, masks = (t.cpu() for t in details[0])
      _equal_bits(masks, _ops.nnm_bits(_ops.nnm_select(raw, f)))
      _within_bound(raw.numpy(), Y.astype(np.float64))   # NNM's "raw" distances are those of the clipped rows
      Y = _np_mix(Y, masks.numpy(), f)
    else:
      assert len(details) == 1
    # the rule on the NumPy-clipped (and mixed) rows: the stand-alone kernel without pre-aggregation gives the same bits
    state_plain = {"center": center_plain} if rule == "centered-clipping" else state
    ref, ref_dist, ref_info = gar_ops.aggregate(plain, torch.from_numpy(Y).cuda(), return_details=True, **state_plain)
    _equal_bits(out, ref)
    _equal_bits(dist, ref_dist)
    _equal_bits(info[:64], ref_info[:64])
    if rule == "dnc":
      _equal_bits(info[96:96 + spec.iterations], ref_info[96:96 + spec.iterations])
    if rule == "centered-clipping":
      _equal_bits(center, center_plain)


def test_fall_backs_match_the_reference():
  from aggregathor_b200.ops import gar as gar_ops
  G = _data(9, 3001, seed=4, outliers=2)
  for mix in ("arc", "arc+nnm"):
    for rule in ("trimmed-mean", "krum", "median"):
      spec = FusedSpec(rule, 9, f=2, m=5 if rule == "krum" else 0, mix=mix)
      out = gar_ops.aggregate(spec, G.double().cuda())
      assert out.dtype == torch.float64
      ref = gar_ops._torch_rules(spec)(_ops.torch_pre_aggregate(G.double(), mix, 2))
      assert float((out.cpu() - ref).abs().max()) <= 1e-12 * max(1.0, float(ref.abs().max()))
    G36 = _data(36, 2001, seed=6, outliers=3)
    out = gar_ops.aggregate(FusedSpec("trimmed-mean", 36, f=5, mix=mix), G36.cuda())
    ref = _ops.torch_trimmed_mean(_ops.torch_pre_aggregate(G36.double(), mix, 5), 5)
    assert float((out.cpu().double() - ref).abs().max()) < 1e-5
    center = torch.zeros(2001, device="cuda")
    out = gar_ops.aggregate(FusedSpec("centered-clipping", 36, f=5, iterations=2, tau=3.0, mix=mix), G36.cuda(), center=center)
    ref = _ops.torch_centered_clipping(_ops.torch_pre_aggregate(G36.double(), mix, 5), 2, 3.0, torch.zeros(2001, dtype=torch.float64))
    assert float((out.cpu().double() - ref).abs().max()) < 1e-5


def test_kernel_rejects_invalid_parameters():
  from aggregathor_b200.ops import gar as gar_ops
  G = torch.randn(8, 64, device="cuda")
  rows = [G.data_ptr() + i * 64 * 4 for i in range(8)]
  for mix in ("arc", "arc+nnm"):
    for rule in ("average", "median", "geometric-median"):
      with pytest.raises(RuntimeError, match="status 120"):
        gar_ops.aggregate(FusedSpec(rule, 8, f=4, mix=mix), G)
    with pytest.raises(RuntimeError, match="status 120"):
      gar_ops.aggregate(FusedSpec("average", 8, f=-1, mix=mix), G)
    launcher = gar_ops.FusedLauncher(G.device, 8)
    out = torch.empty(64, device="cuda")
    staging = torch.empty((8, 64), device="cuda")
    with pytest.raises(RuntimeError, match="status 108"):   # no staging buffer to clip in
      launcher.launch(FusedSpec("average", 8, f=2, mix=mix), rows, 0, 64, agg_out=out)
    krum = FusedSpec("krum", 8, f=2, m=4, mix=mix)
    with pytest.raises(RuntimeError, match="status 111"):   # bucketed phase-A kernels refuse a pre-aggregation
      launcher.phase_a(krum, rows, [(0, 32), (32, 64)], 0, staging=staging)
    with pytest.raises(RuntimeError, match="status 111"):   # nothing may be pre-accumulated
      launcher.launch(krum, rows, segments=[(0, 32), (32, 64)], agg_out=out, staging=staging, first_seg=1)
  torch.cuda.synchronize()


def _manager(rule, engine, attack, mix, args=(), k=2, n=8):
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate(rule, n, k, list(args))
  return Manager(experiment, gar, n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cuda", engine=engine, seed=7,
                 attack=attacks.instantiate(attack, n, k, []), nb_real_byz=k, worker_momentum=0.9, worker_momentum_dampening=0.1,
                 pre_aggregation=mix, nb_decl_byz=k)


@pytest.mark.parametrize("mix", ["arc", "arc+nnm"])
@pytest.mark.parametrize("attack", ["alie", "flip"])
@pytest.mark.parametrize("rule,args", [("trimmed-mean", []), ("krum", []), ("centered-clipping", ["iterations:3", "tau:1"]), ("median", []),
                                       ("dnc", ["subsample:5000"])])
def test_fused_engine_matches_the_baseline_engine(rule, args, attack, mix):
  fused = _manager(rule, "fused", attack, mix, args)
  base = _manager(rule, "baseline", attack, mix, args)
  assert fused.aggregation.name == "fused" and base.aggregation.name == "baseline"
  assert fused.aggregation.spec.mix == mix and fused.aggregation.staging is not None
  for _ in range(3):
    fused.train()
    base.train()
    torch.cuda.synchronize()
  _equal_bits(fused.params, base.params)
  if rule == "centered-clipping":
    _equal_bits(fused.aggregation.center, base.aggregation.center)
  assert bool(torch.isfinite(fused.params).all())
  fused.close()
  base.close()


def test_no_bucketed_overlap_with_arc(monkeypatch):
  monkeypatch.setenv("AGB_OVERLAP", "2")
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate("krum", 8, 2, [])
  mgr = Manager(experiment, gar, 8, "sgd", [], "fixed", ["initial-rate:0.05"], device="cuda", engine="fused", pre_aggregation="arc")
  assert len(mgr.aggregation.buckets) == 1 and not mgr.aggregation.overlappable and not mgr._bucket_layers
  mgr.train()
  assert bool(torch.isfinite(mgr.params).all())
  mgr.close()


def _gpus():
  return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_gpus() < 2, reason="needs at least 2 GPUs")
@pytest.mark.parametrize("mix", ["arc", "arc+nnm"])
def test_fused_matches_baseline_on_all_ranks(tmp_path, mix):
  nproc = max(r for r in range(1, min(_gpus(), 8) + 1) if 8 % r == 0)
  port = 29600 + os.getpid() % 90
  rules = "trimmed-mean,krum,bulyan,centered-clipping,average,dnc"
  cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1", "--master-port", str(port),
         str(ROOT / "benchmarks" / "gar_bench.py"), "--gar-dim", "1000003", "--gar-iters", "3", "--gar-rules", rules, "--gar-pre-aggregation", mix,
         "--gar-out", str(tmp_path)]
  proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=900, cwd=str(ROOT))
  out = proc.stdout.decode(errors="replace")
  assert proc.returncode == 0, out[-4000:]
  results = json.loads((tmp_path / ("gar_bench_%d.json" % nproc)).read_text())["results"]
  for rule in rules.split(","):
    entry = results[rule]
    assert entry["pre_aggregation"] == mix
    assert entry["replicas_identical"], entry
    assert entry["max_abs_diff_vs_baseline"] < 1e-4, entry

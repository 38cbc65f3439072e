"""sm_90a bucketing inside the aggregation kernel: every rule replayed bit for bit on NumPy bucket means (NaN and infinite rows
included), the kernel's permutation and masks against `_ops`, the status codes, fused (CUDA graph, device step key) vs baseline
training with worker momentum under ALIE and flip, SMEA at (32, 4), and the multi-GPU engine."""

import ctypes
import json
import math
import os
import pathlib
import subprocess
import sys

import numpy as np
import pytest
import torch

from aggregathor_b200 import aggregators, attacks, experiments, tools
from aggregathor_b200.aggregators import FusedSpec, _ops
from aggregathor_b200.engine.trainer import Manager

pytestmark = pytest.mark.gpu
ROOT = pathlib.Path(__file__).resolve().parent.parent
RULES = ["average", "average-nan", "median", "averaged-median", "krum", "bulyan", "trimmed-mean", "mda", "geometric-median",
         "centered-clipping", "dnc", "smea"]


def _data(n, d, seed):
  gen = torch.Generator().manual_seed(seed)
  G = torch.randn(n, d, generator=gen)
  G[n - 1] = G[n - 1] * 30 + 5
  if n >= 8:   # a few NaNs in row 0, infinities of both signs in rows 1 and 2
    G[0, 3::211] = float("nan")
    G[1, 5::307] = float("inf")
    G[2, 5::613] = float("-inf")
  return G


def _equal_bits(a, b):
  a, b = torch.as_tensor(a).cpu(), torch.as_tensor(b).cpu()
  assert a.dtype == b.dtype and a.shape == b.shape
  nan = torch.isnan(a)
  assert torch.equal(nan, torch.isnan(b))
  diff = (a[~nan].view(torch.int32) != b[~nan].view(torch.int32)).nonzero()
  assert diff.numel() == 0, (int(diff[0]), float(a[~nan][diff[0]]), float(b[~nan][diff[0]]))


def _np_means(X, masks):
  """Bucket means in NumPy fp32: members added in ascending worker order from +0, one division."""
  out = []
  with np.errstate(over="ignore", invalid="ignore"):
    for mask in masks:
      members = [j for j in range(X.shape[0]) if (int(mask) & 0xffffffff) >> j & 1]
      acc = np.zeros(X.shape[1], dtype=np.float32)
      for j in members:
        acc = acc + X[j]
      out.append(acc / np.float32(len(members)))
  return np.stack(out).astype(np.float32)


def _spec(rule, rows, s):
  """The rule for `rows` bucket means with the largest f it accepts there (at most 2), or None."""
  kwargs = {"geometric-median": dict(iterations=3), "centered-clipping": dict(iterations=3, tau=2.0),
            "dnc": dict(iterations=2, subsample=700, seed=5)}.get(rule, {})
  for f in (2, 1, 0):
    if rule in ("krum", "bulyan", "trimmed-mean", "mda", "geometric-median", "centered-clipping", "dnc", "smea") and 2 * f >= rows:
      continue
    if rule == "krum" and rows - f - 2 < 1:
      continue
    if rule == "bulyan" and (f < 1 or rows < 4 * f + 3):
      continue
    if rule == "smea" and math.comb(rows, f) > _ops.SMEA_MAX_SETS:
      continue
    m = rows - f - 2 if rule in ("krum", "bulyan") else 0
    beta = rows - 4 * f - 2 if rule == "bulyan" else (max(1, rows - f) if rule == "averaged-median" else 0)
    return FusedSpec(rule, rows, f=f, m=m, beta=beta, mix="bucketing", bucket_size=s, **kwargs)
  return None


@pytest.mark.parametrize("s", [1, 2, 3, "n"])
@pytest.mark.parametrize("n", [3, 8, 9, 17, 32])
@pytest.mark.parametrize("rule", RULES)
def test_kernel_replays_bit_for_bit(rule, n, s):
  from aggregathor_b200.ops import gar as gar_ops
  s = n if s == "n" else s
  if s > n:
    pytest.skip("s > n")
  rows = _ops.check_bucketing(n, s)
  if rule in ("krum", "bulyan", "mda", "smea", "dnc") and rows < 3:
    pytest.skip("the selection rules' own GPU tests start at n = 3")
  spec = _spec(rule, rows, s)
  if spec is None:
    pytest.skip("%s is not valid at n' = %d" % (rule, rows))
  plain = spec.with_mix(None)
  d = 2003
  calls = 2 if rule in ("centered-clipping", "dnc") else 1
  center, center_plain = torch.zeros(d, device="cuda"), torch.zeros(d, device="cuda")
  for call in range(calls):
    step = 3 + 5 * call
    G = _data(n, d, seed=n * 13 + len(rule) + s + call)
    state = {"center": center} if rule == "centered-clipping" else {}
    out, dist, info, *details = gar_ops.aggregate(spec, G.cuda(), return_details=True, step=step, bucketing_seed=17, **state)
    if rule == "smea":
      details = details[1:]
    assert len(details) == 1
    perm, masks = (t.cpu() for t in details[0])
    _, perm_ref, masks_ref = _ops.torch_bucketing(G, s, 17, step, return_details=True)
    _equal_bits(perm, perm_ref)
    _equal_bits(masks, masks_ref)
    Y = _np_means(G.numpy(), masks.tolist())
    # the rule on the NumPy bucket means: the stand-alone kernel without pre-aggregation gives the same bits
    state_plain = {"center": center_plain} if rule == "centered-clipping" else {}
    ref = gar_ops.aggregate(plain, torch.from_numpy(Y).cuda(), return_details=True, step=step, **state_plain)
    # the two calls run on different cached launchers: compare the details the rule writes, not what earlier calls left in them
    _equal_bits(out, ref[0])
    if rule in ("krum", "bulyan", "mda", "smea", "dnc", "geometric-median", "centered-clipping"):
      _equal_bits(dist, ref[1])
    if rule in ("krum", "bulyan", "mda", "smea", "dnc"):   # theta, then the selection masks
      theta = int(ref[2][0])
      _equal_bits(info[:1 + theta], ref[2][:1 + theta])
    if rule == "dnc":
      _equal_bits(info[96:96 + spec.iterations], ref[2][96:96 + spec.iterations])
    if rule == "centered-clipping":
      _equal_bits(center, center_plain)


def test_step_changes_the_permutation_and_fall_backs():
  from aggregathor_b200.ops import gar as gar_ops
  G = _data(16, 1001, seed=3)
  spec = FusedSpec("average", 8, mix="bucketing", bucket_size=2)
  perms = set()
  for step in (1, 2, 3):
    out, _, _, (perm, masks) = gar_ops.aggregate(spec, G.cuda(), return_details=True, step=step)
    perms.add(tuple(perm.tolist()))
    _equal_bits(out, gar_ops.aggregate(FusedSpec("average", 8), _ops.torch_bucketing(G, 2, 0, step).cuda()))
  assert len(perms) == 3
  # float64 and more than 32 rows: the torch reference on the device
  G9 = G[:9].nan_to_num(0.0, 0.0, 0.0).double()   # finite rows: a tolerance, since the device and the host reduce in other orders
  out = gar_ops.aggregate(FusedSpec("trimmed-mean", 5, f=1, mix="bucketing", bucket_size=2), G9.cuda(), step=4)
  ref = _ops.torch_trimmed_mean(_ops.torch_bucketing(G9, 2, 0, 4), 1)
  assert out.dtype == torch.float64 and float((out.cpu() - ref).abs().max()) <= 1e-12 * max(1.0, float(ref.abs().max()))
  G40 = _data(40, 501, seed=8)
  out = gar_ops.aggregate(FusedSpec("median", 20, mix="bucketing", bucket_size=2), G40.cuda(), step=6)
  _equal_bits(out, _ops.torch_median(_ops.torch_bucketing(G40.cuda(), 2, 0, 6)))


def test_kernel_rejects_invalid_bucketing_arguments():
  from aggregathor_b200.ops import gar as gar_ops
  G = torch.randn(8, 64, device="cuda")
  rows = [G.data_ptr() + i * 64 * 4 for i in range(8)]
  launcher = gar_ops.FusedLauncher(G.device, 8)
  out = torch.empty(64, device="cuda")
  staging = torch.empty((8, 64), device="cuda")
  spec = FusedSpec("average", 4, mix="bucketing", bucket_size=2)
  with pytest.raises(RuntimeError, match="status 123"):   # no staging tile for the means
    launcher.launch(spec, rows, 0, 64, agg_out=out)
  with pytest.raises(RuntimeError, match="status 123"):   # s > n_rows (the spec's own check bypassed)
    bad = FusedSpec("average", 1, mix="bucketing", bucket_size=2)
    launcher.launch(bad, rows[:1], 0, 64, agg_out=out, staging=staging)
  # argument blocks FusedSpec never produces, patched after `_fill`: bucketing with NNM or ARC, and n != ceil(n_rows / s)
  for field, value in (("mix", FusedSpec.MIX_BUCKETING | FusedSpec.MIX_NNM), ("mix", FusedSpec.MIX_BUCKETING | FusedSpec.MIX_ARC), ("n", 5)):
    args, scratch_elems = launcher._fill(spec, rows, [(0, 64)], agg_out=out, staging=staging)
    setattr(args, field, value)
    with pytest.raises(RuntimeError, match="status 123"):
      gar_ops._check(gar_ops._lib().agb_gar_fused(ctypes.byref(args), 0, ctypes.c_longlong(scratch_elems), gar_ops._stream_ptr()), "gar_fused")
  with pytest.raises(tools.UserException, match="reduces 8 gradient rows to 4"):
    launcher.launch(FusedSpec("average", 3, mix="bucketing", bucket_size=2), rows, 0, 64, agg_out=out, staging=staging)
  krum = FusedSpec("krum", 4, f=0, m=1, mix="bucketing", bucket_size=2)
  with pytest.raises(RuntimeError, match="status 111"):   # bucketed phase-A kernels refuse a pre-aggregation
    launcher.phase_a(krum, rows, [(0, 32), (32, 64)], 0, staging=staging)
  with pytest.raises(RuntimeError, match="status 111"):   # nothing may be pre-accumulated
    launcher.launch(krum, rows, segments=[(0, 32), (32, 64)], agg_out=out, staging=staging, first_seg=1)
  torch.cuda.synchronize()


def test_smea_32_4_runs_with_bucketing_only():
  from aggregathor_b200.ops import gar as gar_ops
  G = _data(32, 3001, seed=12)
  with pytest.raises(RuntimeError, match="status 122"):
    gar_ops.aggregate(FusedSpec("smea", 32, f=4), G.cuda())
  spec = FusedSpec("smea", 16, f=4, mix="bucketing", bucket_size=2)
  out, dist, info, score, (perm, masks) = gar_ops.aggregate(spec, G.cuda(), return_details=True, step=9)
  Y = _ops.torch_bucketing(G, 2, 0, 9)
  ids = _ops.smea_select(dist.cpu(), 4)
  good = np.zeros(16, dtype=bool)
  good[ids.numpy()] = True
  _equal_bits(out, _ops.selection_mean(Y, good))
  _equal_bits(out, gar_ops.aggregate(FusedSpec("smea", 16, f=4), Y.cuda()))


def _manager(rule, engine, attack, rows, args=(), k=2, n=8, s=2):
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate(rule, rows, k, list(args))
  return Manager(experiment, gar, n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cuda", engine=engine, seed=7,
                 attack=attacks.instantiate(attack, n, k, []), nb_real_byz=k, worker_momentum=0.9, worker_momentum_dampening=0.1,
                 pre_aggregation="bucketing", bucket_size=s, bucketing_seed=11)


@pytest.mark.parametrize("attack", ["alie", "flip"])
@pytest.mark.parametrize("rule,args,k", [("trimmed-mean", [], 1), ("krum", [], 1), ("centered-clipping", ["iterations:3", "tau:1"], 1),
                                         ("median", [], 1), ("dnc", ["subsample:5000"], 1), ("average", [], 2)])
def test_fused_engine_matches_the_baseline_engine(rule, args, k, attack):
  fused = _manager(rule, "fused", attack, 4, args, k=k)
  base = _manager(rule, "baseline", attack, 4, args, k=k)
  assert fused.aggregation.name == "fused" and base.aggregation.name == "baseline"
  assert fused.aggregation.spec.mix == "bucketing" and fused.aggregation.staging.shape[0] == 4
  assert fused.aggregation.step_dev is not None   # the device step key graph replays read
  perms = set()
  for _ in range(4):
    fused.train()
    base.train()
    torch.cuda.synchronize()
    perms.add(tuple(fused.aggregation.launcher.info[128:136].tolist()))
    _equal_bits(fused.params, base.params)
  assert len(perms) > 1   # replays draw new permutations
  if rule == "centered-clipping":
    _equal_bits(fused.aggregation.center, base.aggregation.center)
  assert bool(torch.isfinite(fused.params).all())
  fused.close()
  base.close()


def test_no_bucketed_overlap_with_bucketing(monkeypatch):
  monkeypatch.setenv("AGB_OVERLAP", "2")
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate("krum", 4, 1, [])
  mgr = Manager(experiment, gar, 8, "sgd", [], "fixed", ["initial-rate:0.05"], device="cuda", engine="fused", pre_aggregation="bucketing",
                bucket_size=2)
  assert len(mgr.aggregation.buckets) == 1 and not mgr.aggregation.overlappable and not mgr._bucket_layers
  mgr.train()
  assert bool(torch.isfinite(mgr.params).all())
  mgr.close()


def _gpus():
  return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_gpus() < 2, reason="needs at least 2 GPUs")
def test_fused_matches_baseline_on_all_ranks(tmp_path):
  nproc = max(r for r in range(1, min(_gpus(), 8) + 1) if 8 % r == 0)
  port = 29700 + os.getpid() % 90
  rules = "trimmed-mean,krum,centered-clipping,average,dnc"
  cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1", "--master-port", str(port),
         str(ROOT / "benchmarks" / "gar_bench.py"), "--gar-dim", "1000003", "--gar-iters", "3", "--gar-rules", rules, "--gar-byz", "1",
         "--gar-pre-aggregation", "bucketing", "--gar-bucket-size", "2", "--gar-out", str(tmp_path)]
  proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=900, cwd=str(ROOT))
  out = proc.stdout.decode(errors="replace")
  assert proc.returncode == 0, out[-4000:]
  results = json.loads((tmp_path / ("gar_bench_%d.json" % nproc)).read_text())["results"]
  for rule in rules.split(","):
    entry = results[rule]
    assert entry["pre_aggregation"] == "bucketing" and entry["rule_rows"] == 4
    assert entry["replicas_identical"], entry
    assert entry["max_abs_diff_vs_baseline"] < 1e-4, entry

"""sm_90a SMEA: the selection and output replayed bit for bit by `_ops` on the kernel's own distance matrix (every pre-aggregation, with
NaN and infinite rows), the float64 covariance oracle at d ~ 1e5, fused vs baseline training under graph replay with worker momentum and
an attack, the bucketed distance pass, the fall-backs, status 122, `gar_bench.py` and the multi-GPU engine."""

import itertools
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
U = 2.0 ** -24
# (n, f) of the replays: f as large as the cap allows where the NumPy replay stays quick (C(17, 3) = 680, C(32, 2) = 496 sets)
CASES = [(3, 1), (8, 2), (9, 4), (17, 3), (32, 2)]


def _data(n, d, seed, outliers=0, non_finite=False):
  gen = torch.Generator().manual_seed(seed)
  G = torch.randn(n, d, generator=gen)
  for k in range(outliers):
    G[n - 1 - k] = G[n - 1 - k] * 30 + 5
  if non_finite:
    G[0, 3::11] = float("nan")
    G[1, 5::13] = float("inf")
  return G


def _equal_bits(a, b):
  a, b = a.cpu(), b.cpu()
  assert a.dtype == b.dtype and a.shape == b.shape
  nan = torch.isnan(a)
  assert torch.equal(nan, torch.isnan(b))
  diff = (a[~nan] != b[~nan]).nonzero()
  assert diff.numel() == 0, (int(diff[0]), float(a[~nan][diff[0]]), float(b[~nan][diff[0]]))


def _mask_ids(info, n):
  mask = int(info[1].item()) & 0xffffffff
  return [i for i in range(n) if (mask >> i) & 1]


def _replayed_rows(G, mix, f, details):
  """The rows the rule saw, rebuilt from the kernel's pre-aggregation details: ARC's factors, then NNM's neighbourhoods."""
  Y = G
  details = list(details)
  nnm = details.pop(0) if mix in ("nnm", "arc+nnm") else None
  if mix in ("arc", "arc+nnm"):
    Y = _ops.torch_arc_clip(Y, details.pop(0)[1].cpu())
  if nnm is not None:
    Y = _ops.torch_nnm_mix(Y, nnm[1].cpu(), f)
  return Y


@pytest.mark.parametrize("non_finite", [False, True])
@pytest.mark.parametrize("mix", FusedSpec.MIXES)
@pytest.mark.parametrize("n,f", CASES)
def test_kernel_replays_bit_for_bit(n, f, mix, non_finite):
  from aggregathor_b200.ops import gar as gar_ops
  G = _data(n, 1003, seed=n * 17 + f, outliers=f if n > 3 else 0, non_finite=non_finite)
  out, dist, info, score, *mixed = gar_ops.aggregate(FusedSpec("smea", n, f=f, mix=mix), G.cuda(), return_details=True)
  assert int(info[0].item()) == 1 and score.dtype == torch.float64
  ids, expect_score = _ops.smea_select(dist.cpu(), f, return_score=True)
  assert _mask_ids(info, n) == ids.tolist(), (n, f, mix)
  assert np.float64(float(score)).view(np.int64) == np.float64(expect_score).view(np.int64)
  good = np.zeros(n, dtype=bool)
  good[ids.numpy()] = True
  _equal_bits(out, _ops.selection_mean(_replayed_rows(G, mix, f, mixed), good))
  if non_finite and mix is None and n > 3:   # rows 0 (NaN) and 1 (inf) are never kept while a finite set exists (n = 3 has none)
    assert 0 not in ids.tolist() and 1 not in ids.tolist()


def test_float64_covariance_oracle_at_large_d():
  from aggregathor_b200.ops import gar as gar_ops
  n, f, d = 8, 2, 100003
  G = _data(n, d, seed=21)
  G[n - 1] += 0.5   # two rows shifted apart along the all-ones direction
  G[n - 2] -= 0.5
  _, dist, info, score = gar_ops.aggregate(FusedSpec("smea", n, f=f), G.cuda(), return_details=True)
  X = G.double().numpy()
  sets = list(itertools.combinations(range(n), n - f))
  lam = []
  for S in sets:
    Y = X[list(S)] - X[list(S)].mean(axis=0)
    lam.append(float(np.linalg.eigvalsh(Y @ Y.T / len(S))[-1]))   # the nonzero spectrum of the covariance
  lam = np.array(lam)
  # the kernel's fp32 distances are within a relative (d + 2) u of float64 in any summation order: B_S moves by at most 2 max|dD| per
  # entry, score / m by 2 (d + 2) u max D
  bound = 2 * (d + 2) * U * float(dist.max()) + 1e-12 * float(lam.max())
  ids = _mask_ids(info, n)
  chosen = sets.index(tuple(ids))
  assert abs(float(score) / (n - f) - lam[chosen]) <= bound
  order = np.argsort(lam, kind="stable")
  if lam[order[1]] - lam[order[0]] > 2 * bound:
    assert chosen == order[0]
  assert lam[chosen] - lam[order[0]] <= 2 * bound
  assert ids == list(range(n - f))   # the two shifted rows are left out


def _manager(engine, **kwargs):
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate("smea", 8, 2, [])
  attack = attacks.instantiate("alie", 8, 2, [])
  return Manager(experiment, gar, 8, "sgd", [], "fixed", ["initial-rate:0.05"], device="cuda", engine=engine, seed=3, attack=attack,
                 nb_real_byz=2, worker_momentum=0.9, worker_momentum_dampening=0.1, **kwargs)


def test_fused_matches_baseline_under_graph_replay_with_momentum_and_alie():
  fused = _manager("fused")
  base = _manager("baseline")
  losses = []
  for _ in range(5):
    losses.append(float(fused.train()))
    base.train()
  torch.cuda.synchronize()
  assert fused._graph is not None   # the workers' passes replay a graph; with an attack the aggregation runs after it
  _equal_bits(fused.params, base.params)
  assert all(np.isfinite(losses))
  fused.close()
  base.close()


def test_fused_engine_matches_the_baseline_engine_under_graph_replay():
  from aggregathor_b200.parallel.aggregation import BaselineAggregation, FusedAggregation
  n, f = 8, 2
  layout = FlatLayout()
  layout.add("w", (1000, 37))
  layout.add("b", (37,))
  layout.freeze()
  gar = aggregators.instantiate("smea", n, f, [])
  fused = FusedAggregation(gar, layout, n, build(optimizers, "optimizer", "sgd", []), device="cuda", keep_aggregate=True, device_state=True)
  base = BaselineAggregation(gar, layout, n, build(optimizers, "optimizer", "sgd", []), device="cuda")
  d = layout.padded_size
  init = torch.randn(d, generator=torch.Generator().manual_seed(1)).cuda()
  fused.params.copy_(init)
  base.params.copy_(init)
  grads = [_data(n, d, seed=10 + k, outliers=f).cuda() for k in range(4)]
  fused.grads.copy_(grads[0])
  fused.step(0.1)
  base.grads.copy_(grads[0])
  base.step(0.1)
  graph = torch.cuda.CUDAGraph()
  fused.prepare(0.1)
  fused.grads.copy_(grads[1])
  torch.cuda.synchronize()
  with torch.cuda.graph(graph, stream=torch.cuda.Stream()):
    fused.step(prepared=True)
  graph.replay()
  base.grads.copy_(grads[1])
  base.step(0.1)
  for k in (2, 3):
    fused.prepare(0.1)
    fused.grads.copy_(grads[k])
    graph.replay()
    base.grads.copy_(grads[k])
    base.step(0.1)
    torch.cuda.synchronize()
    _equal_bits(fused.last_aggregate, base.last_aggregate)
    _equal_bits(fused.params, base.params)
    assert _mask_ids(fused.launcher.info, n) == list(range(n - f))


@pytest.mark.parametrize("n,f", [(8, 2), (11, 3), (20, 2)])
def test_bucketed_phase_a_matches_the_single_launch(n, f):
  from aggregathor_b200.parallel.aggregation import FusedAggregation
  layout = FlatLayout()
  layout.add("a", (3000, 11))
  layout.add("b", (513,))
  layout.add("c", (77, 64))
  layout.freeze()
  d = layout.padded_size
  gar = aggregators.instantiate("smea", n, f, [])
  cut1, cut2 = (2 * d // 3) // 8 * 8, (d // 4) // 8 * 8
  plain = FusedAggregation(gar, layout, n, build(optimizers, "optimizer", "sgd", []), device="cuda", keep_aggregate=True)
  bucketed = FusedAggregation(gar, layout, n, build(optimizers, "optimizer", "sgd", []), device="cuda", keep_aggregate=True,
                              buckets=[(cut1, d), (cut2, cut1), (0, cut2)], device_state=True)
  assert bucketed.overlappable and len(bucketed.segments) == 3
  gen = torch.Generator().manual_seed(9)
  init = torch.randn(d, generator=gen)
  plain.params.copy_(init)
  bucketed.params.copy_(init)
  side = torch.cuda.Stream()
  for step in range(3):
    G = torch.randn(n, d, generator=gen) * 0.1
    G[n - f:] += 2.0
    plain.grads.copy_(G)
    bucketed.grads.copy_(G)
    plain.step(0.1)
    bucketed.prepare(0.1)
    side.wait_stream(torch.cuda.current_stream())
    bucketed.phase_a(0, stream=side)
    bucketed.phase_a(1, stream=side)
    torch.cuda.current_stream().wait_stream(side)
    bucketed.step(prepared=True)
    torch.cuda.synchronize()
    assert torch.equal(plain.launcher.info[:2], bucketed.launcher.info[:2])
    assert _mask_ids(plain.launcher.info, n) == list(range(n - f))
    assert _mask_ids(bucketed.launcher.info, n) == _ops.smea_select(bucketed.launcher.dist_out.view(n, n).cpu(), f).tolist()
    _equal_bits(bucketed.last_aggregate, plain.last_aggregate)
    _equal_bits(bucketed.params, plain.params)


def test_double_inputs_and_more_than_32_workers_fall_back():
  from aggregathor_b200.ops import gar as gar_ops
  G = _data(9, 3001, seed=4, outliers=2).double()
  out = gar_ops.aggregate(FusedSpec("smea", 9, f=2), G.cuda())
  assert out.dtype == torch.float64
  assert torch.equal(out.cpu(), _ops.torch_smea(G, 2))
  G = _data(36, 2001, seed=6, outliers=2)
  out = gar_ops.aggregate(FusedSpec("smea", 36, f=2, mix="nnm"), G.cuda())
  _equal_bits(out, _ops.torch_smea(_ops.torch_pre_aggregate(G.cuda(), "nnm", 2), 2))
  gar = aggregators.instantiate("smea", 8, 2, [])
  G = _data(8, 3000, seed=11, outliers=2).cuda()
  _equal_bits(gar.aggregate(list(G)), gar_ops.aggregate(gar.fused_spec(), G))


def test_kernel_rejects_invalid_parameters():
  from aggregathor_b200.ops import gar as gar_ops
  G = torch.randn(32, 64, device="cuda")
  for n, f in ((8, 4), (8, -1), (32, 4), (21, 5)):   # 2 f >= n, f < 0, C(32, 4) = 35960 and C(21, 5) = 20349 > 2^14
    with pytest.raises(RuntimeError, match="status 122"):
      gar_ops.aggregate(FusedSpec("smea", n, f=f), G[:n])


def test_gar_bench_runs_smea(tmp_path):
  cmd = [sys.executable, str(ROOT / "benchmarks" / "gar_bench.py"), "--gar-dim", "200003", "--gar-iters", "3", "--gar-rules", "krum,smea",
         "--gar-out", str(tmp_path)]
  proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, cwd=str(ROOT))
  out = proc.stdout.decode(errors="replace")
  assert proc.returncode == 0, out[-4000:]
  entry = json.loads((tmp_path / "gar_bench_1.json").read_text())["results"]["smea"]
  assert entry["replicas_identical"] and entry["max_abs_diff_vs_baseline"] == 0.0, entry


def _gpus():
  return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_gpus() < 2, reason="needs at least 2 GPUs")
def test_fused_matches_baseline_on_all_ranks(tmp_path):
  nproc = max(r for r in range(1, min(_gpus(), 8) + 1) if 8 % r == 0)
  port = 29700 + os.getpid() % 90
  cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1", "--master-port", str(port),
         str(ROOT / "benchmarks" / "gar_bench.py"), "--gar-dim", "1000003", "--gar-iters", "3", "--gar-rules", "smea", "--gar-out", str(tmp_path)]
  proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, cwd=str(ROOT))
  out = proc.stdout.decode(errors="replace")
  assert proc.returncode == 0, out[-4000:]
  entry = json.loads((tmp_path / ("gar_bench_%d.json" % nproc)).read_text())["results"]["smea"]
  assert entry["replicas_identical"], entry
  assert entry["max_abs_diff_vs_baseline"] < 1e-4, entry

"""sm_90a trimmed mean and MDA against the host library: bit-exact coordinate pass, MDA selection checked on the kernel's own
distance matrix, the fused engine with every optimizer, the bucketed distance pass, plug-in dispatch and the multi-GPU engine."""

import json
import math
import os
import pathlib
import subprocess
import sys

import pytest
import torch

from aggregathor_b200 import aggregators
from aggregathor_b200.aggregators import FusedSpec, _ops
from aggregathor_b200.engine.flat import FlatLayout
from aggregathor_b200.engine.optimizers import optimizers
from aggregathor_b200.engine.schedules import build

pytestmark = pytest.mark.gpu
ROOT = pathlib.Path(__file__).resolve().parent.parent
WORKERS = [5, 8, 11, 16, 19, 24, 32]


def _data(n, d, seed, outliers=0, non_finite=False):
  gen = torch.Generator().manual_seed(seed)
  G = torch.randn(n, d, generator=gen)
  for k in range(outliers):
    G[n - 1 - k] = G[n - 1 - k] * 30 + 5
  if non_finite:
    G[0, 3::11] = float("nan")
    G[1, 5::13] = float("inf")
    G[2 % n, 7::17] = float("-inf")
    G[:, 1] = float("nan")          # every value of one coordinate
  return G


def _equal_bits(a, b):
  a, b = a.cpu(), b.cpu()
  assert a.dtype == b.dtype and a.shape == b.shape
  nan = torch.isnan(a)
  assert torch.equal(nan, torch.isnan(b))
  diff = (a[~nan] != b[~nan]).nonzero()
  assert diff.numel() == 0, (int(diff[0]), float(a[~nan][diff[0]]), float(b[~nan][diff[0]]))


def _ordered_mean(G, ids):
  """fp32 mean of rows `ids` added in ascending order from zero, then divided once: the host's `selection_mean`."""
  acc = torch.zeros(G.shape[1], dtype=G.dtype)
  for i in sorted(ids):
    acc = acc + G[i]
  return acc / len(ids)


def _largest_f(n):
  return max(f for f in range(n) if 2 * f < n and math.comb(n, f) <= _ops.MDA_MAX_SETS)


def _mask_ids(info, n):
  mask = int(info[1].item()) & 0xffffffff
  return [i for i in range(n) if (mask >> i) & 1]


@pytest.mark.parametrize("d", [4096, 1003])
@pytest.mark.parametrize("n", WORKERS)
def test_trimmed_mean_bit_exact(n, d):
  from aggregathor_b200.ops import gar as gar_ops
  G = _data(n, d, seed=n * 13 + d, outliers=2, non_finite=True)
  for f in sorted({0, 1, n // 4, (n - 1) // 2}):
    out = gar_ops.aggregate(FusedSpec("trimmed-mean", n, f=f), G.cuda())
    _equal_bits(out, _ops.host_trimmed_mean(G, f))


@pytest.mark.parametrize("d", [4096, 1003])
@pytest.mark.parametrize("n", WORKERS)
def test_mda_selection_and_mean(n, d):
  from aggregathor_b200.ops import gar as gar_ops
  for f in sorted({1, _largest_f(n)}):
    G = _data(n, d, seed=n * 7 + f + d, outliers=f)
    out, dist, info = gar_ops.aggregate(FusedSpec("mda", n, f=f), G.cuda(), return_details=True)
    assert int(info[0].item()) == 1
    ids = _mask_ids(info, n)
    assert ids == _ops.host_mda_select(dist.cpu(), f).tolist(), (n, f)
    _equal_bits(out, _ordered_mean(G, ids))
    # well-separated data: the host, on its own distances, selects the same set (the honest rows)
    _, host_ids = _ops.host_mda(G, f, return_selected=True)
    assert ids == host_ids.tolist() == list(range(n - f))


def test_mda_envelope_worst_case():
  """n = 32, f = 6: the 906192 removal sets of the largest supported search."""
  from aggregathor_b200.ops import gar as gar_ops
  n, f = 32, 6
  G = _data(n, 777, seed=5)   # no outliers: the diameters of many sets are close, the search has to be exact
  out, dist, info = gar_ops.aggregate(FusedSpec("mda", n, f=f), G.cuda(), return_details=True)
  ids = _mask_ids(info, n)
  assert len(ids) == n - f
  assert ids == _ops.host_mda_select(dist.cpu(), f).tolist()
  assert ids == _ops.host_mda_select(dist.cpu().double(), f).tolist()
  _equal_bits(out, _ordered_mean(G, ids))
  # six outliers among 32 rows: the kernel and the host, each on its own distances, keep the same 26 rows
  G = _data(n, 777, seed=6, outliers=f)
  out, _, info = gar_ops.aggregate(FusedSpec("mda", n, f=f), G.cuda(), return_details=True)
  _, host_ids = _ops.host_mda(G, f, return_selected=True)
  assert _mask_ids(info, n) == host_ids.tolist() == list(range(n - f))
  _equal_bits(out, _ops.host_mda(G, f))


@pytest.mark.parametrize("values,f,expected", [
  ([0.0, 1.0, 2.0, 3.0], 1, [0, 1, 2]),
  ([5.0, 0.0, 10.0, 0.0, 10.0], 2, [0, 1, 3]),
  ([10.0, 0.0, 10.0, 0.0, 5.0], 2, [0, 2, 4]),
  ([0.0, 10.0, 5.0, 10.0, 0.0], 2, [0, 2, 4]),
])
def test_mda_kernel_tie_break(values, f, expected):
  """Integer points on a line: exact distances with tied diameters; the lexicographically smallest kept set wins."""
  from aggregathor_b200.ops import gar as gar_ops
  G = torch.tensor(values).unsqueeze(1).repeat(1, 4)
  _, _, info = gar_ops.aggregate(FusedSpec("mda", len(values), f=f), G.cuda(), return_details=True)
  assert _mask_ids(info, len(values)) == expected
  E = torch.eye(12)   # pairwise equidistant rows: every set ties
  _, _, info = gar_ops.aggregate(FusedSpec("mda", 12, f=3), E.cuda(), return_details=True)
  assert _mask_ids(info, 12) == list(range(9))


def test_mda_kernel_excludes_non_finite_rows():
  from aggregathor_b200.ops import gar as gar_ops
  G = _data(11, 3001, seed=2)
  G[4, 10] = float("nan")
  G[7, :] = float("inf")
  out, _, info = gar_ops.aggregate(FusedSpec("mda", 11, f=2), G.cuda(), return_details=True)
  ids = _mask_ids(info, 11)
  assert 4 not in ids and 7 not in ids and bool(torch.isfinite(out).all())
  _equal_bits(out, _ops.host_mda(G, 2))


@pytest.mark.parametrize("rule", ["trimmed-mean", "mda"])
def test_double_precision_inputs_stay_double(rule):
  from aggregathor_b200.ops import gar as gar_ops
  n, f = 9, 2
  G = _data(n, 3001, seed=4, outliers=f).double()
  G += torch.randn(G.shape, generator=torch.Generator().manual_seed(1), dtype=torch.float64) * 1e-9
  out = gar_ops.aggregate(FusedSpec(rule, n, f=f), G.cuda())
  ref = _ops.torch_trimmed_mean(G, f) if rule == "trimmed-mean" else _ops.torch_mda(G, f)
  assert out.dtype == torch.float64
  assert float((out.cpu() - ref).abs().max()) <= 1e-12 * max(1.0, float(ref.abs().max()))


def test_more_than_32_workers_use_the_device_torch_rules():
  from aggregathor_b200.ops import gar as gar_ops
  n, f = 36, 3
  G = _data(n, 2001, seed=6, outliers=f)
  out =gar_ops.aggregate(FusedSpec("trimmed-mean", n, f=f), G.cuda())
  assert float((out.cpu().double() - _ops.torch_trimmed_mean(G.double(), f)).abs().max()) < 1e-5
  out = gar_ops.aggregate(FusedSpec("mda", n, f=f), G.cuda())
  assert float((out.cpu().double() - _ops.torch_mda(G.double(), f)).abs().max()) < 1e-5


@pytest.mark.parametrize("rule", ["trimmed-mean", "mda"])
@pytest.mark.parametrize("opt", ["sgd", "adam", "rmsprop", "adagrad", "adadelta"])
def test_fused_optimizers_single_rank(rule, opt):
  """Fused kernel (R = 1) with every optimizer vs HostAggregation running the same rule on the host and the update in torch."""
  from aggregathor_b200.parallel.aggregation import FusedAggregation, HostAggregation
  layout = FlatLayout()
  layout.add("w", (1000, 37))
  layout.add("b", (37,))
  layout.freeze()
  gar = aggregators.instantiate(rule, 8, 2, [])
  fused = FusedAggregation(gar, layout, 8, build(optimizers, "optimizer", opt, []), device="cuda", keep_aggregate=True)
  host = HostAggregation(gar, layout, 8, build(optimizers, "optimizer", opt, []), device="cpu")
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
    _equal_bits(fused.last_aggregate, host.last_aggregate)
    assert float((fused.params.cpu() - host.params).abs().max()) <= 1e-4 * max(1.0, float(host.params.abs().max()))


@pytest.mark.parametrize("n,f", [(8, 2), (11, 3), (20, 4)])
def test_mda_bucketed_phase_a_matches_the_single_launch(n, f):
  from aggregathor_b200.parallel.aggregation import FusedAggregation
  layout = FlatLayout()
  layout.add("a", (3000, 11))
  layout.add("b", (513,))
  layout.add("c", (77, 64))
  layout.freeze()
  d = layout.padded_size
  gar = aggregators.instantiate("mda", n, f, [])
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
    losses = torch.arange(1, n + 1, dtype=torch.float32, device="cuda") * (step + 1)
    plain.step(0.1, loss_in=losses)
    bucketed.prepare(0.1)
    side.wait_stream(torch.cuda.current_stream())
    bucketed.phase_a(0, stream=side)
    bucketed.phase_a(1, stream=side)
    torch.cuda.current_stream().wait_stream(side)
    bucketed.step(loss_in=losses, prepared=True)
    torch.cuda.synchronize()
    assert int(bucketed.epoch_dev.item()) == step + 1
    assert abs(float(bucketed.loss_out) - float(losses.sum())) < 1e-3
    assert torch.equal(plain.launcher.info[:2], bucketed.launcher.info[:2])
    assert _mask_ids(plain.launcher.info, n) == list(range(n - f))
    assert _mask_ids(bucketed.launcher.info, n) == _ops.host_mda_select(bucketed.launcher.dist_out.view(n, n).cpu(), f).tolist()
    _equal_bits(bucketed.last_aggregate, plain.last_aggregate)
    _equal_bits(bucketed.params, plain.params)


def test_plugin_dispatch_on_cuda():
  G = _data(8, 3000, seed=11, outliers=2)
  for name in ("trimmed-mean", "mda"):
    gar = aggregators.instantiate(name, 8, 2, [])
    _equal_bits(gar.aggregate(list(G.cuda())), gar.aggregate(list(G)))


def test_kernel_rejects_invalid_parameters():
  from aggregathor_b200.ops import gar as gar_ops
  G = torch.randn(32, 64, device="cuda")
  with pytest.raises(RuntimeError, match="invalid MDA parameters"):
    gar_ops.aggregate(FusedSpec("mda", 32, f=7), G)
  with pytest.raises(RuntimeError, match="invalid MDA parameters"):
    gar_ops.aggregate(FusedSpec("mda", 8, f=4), G[:8])
  with pytest.raises(RuntimeError, match="invalid trimmed-mean parameters"):
    gar_ops.aggregate(FusedSpec("trimmed-mean", 8, f=4), G[:8])


def _gpus():
  return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_gpus() < 2, reason="needs at least 2 GPUs")
def test_fused_matches_baseline_on_all_ranks(tmp_path):
  nproc = max(r for r in range(1, min(_gpus(), 8) + 1) if 8 % r == 0)
  port = 29900 + os.getpid() % 90
  cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1", "--master-port", str(port),
         str(ROOT / "benchmarks" / "gar_bench.py"), "--gar-dim", "1000003", "--gar-iters", "3", "--gar-rules", "trimmed-mean,mda", "--gar-out", str(tmp_path)]
  proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, cwd=str(ROOT))
  out = proc.stdout.decode(errors="replace")
  assert proc.returncode == 0, out[-4000:]
  results = json.loads((tmp_path / ("gar_bench_%d.json" % nproc)).read_text())["results"]
  assert set(results) == {"trimmed-mean", "mda"}
  for rule, entry in results.items():
    assert entry["replicas_identical"], (rule, entry)
    assert entry["max_abs_diff_vs_baseline"] < 1e-4, (rule, entry)

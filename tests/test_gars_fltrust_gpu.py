"""FLTrust on the H100: the stand-alone sm_90a kernel against a float64 oracle of its sums and bit for bit against the torch reference fed
those sums, the fused engine against the baseline engine, and whole-step CUDA-graph replays against eager steps."""

import os
import subprocess
import sys
import pathlib

import numpy as np
import pytest
import torch

from aggregathor_b200 import aggregators, attacks, experiments
from aggregathor_b200.aggregators import FusedSpec, _ops

pytestmark = pytest.mark.gpu
ROOT = pathlib.Path(__file__).resolve().parent.parent


def _equal_bits(a, b):
  a, b = a.detach().cpu().contiguous(), b.detach().cpu().contiguous()
  assert a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


def _case(n, d, seed, kind):
  gen = torch.Generator().manual_seed(seed)
  r = torch.randn(d, generator=gen)
  G = 0.3 * r + torch.randn((n, d), generator=gen) * torch.rand((n, 1), generator=gen) * 2
  if kind == "nan" and n > 1:
    G[1, d // 3] = float("nan")
    G[n - 1, 0] = float("inf")
  elif kind == "negative":
    G = -G.abs() * r.sign()
  elif kind == "zero-root":
    r = torch.zeros(d)
  elif kind == "mixed" and n > 2:
    G[::3] *= -1.0
    G[2] *= 100.0
  return G, r


@pytest.mark.parametrize("d", [1003, 40960])
@pytest.mark.parametrize("kind", ["plain", "mixed", "nan", "negative", "zero-root"])
@pytest.mark.parametrize("n", list(range(1, 33)))
def test_standalone_kernel(n, kind, d):
  from aggregathor_b200.ops import gar as gar_ops
  G, r = _case(n, d, 100 * n + d % 7, kind)
  out, P, N, N0, a = gar_ops.aggregate(FusedSpec("fltrust", n), G.cuda(), root=r.cuda(), return_details=True)
  # the sums against float64, where the row is finite
  Gd, rd = G.double().numpy(), r.double().numpy()
  finite = np.isfinite(Gd).all(axis=1)
  absdot = np.abs(Gd[finite]) @ np.abs(rd)
  assert np.all(np.abs(P.numpy()[finite] - Gd[finite] @ rd) <= 1e-5 * absdot + 1e-30)
  assert np.allclose(N.numpy()[finite], (Gd[finite] ** 2).sum(axis=1), rtol=1e-5, atol=0)
  assert abs(float(N0) - float(rd @ rd)) <= 1e-5 * float(rd @ rd)
  assert not np.isfinite(N.numpy()[~finite]).all() if (~finite).any() else True
  # given the kernel's sums, the torch reference produces the same coefficients and the same bits
  ref, *details = _ops.torch_fltrust(G.cuda(), r.cuda(), sums=(P.numpy(), N.numpy(), float(N0)), return_details=True)
  assert np.array_equal(details[3], a.numpy())
  _equal_bits(out, ref)
  if kind in ("negative", "zero-root"):
    assert not a.numpy().any() and torch.equal(out.cpu(), torch.zeros(d)) and not torch.signbit(out.cpu()).any()
  if kind == "nan" and n > 1:
    assert a[1] == 0 and a[n - 1] == 0 and bool(torch.isfinite(out).all())
  assert float(torch.linalg.norm(out.double())) <= float(torch.linalg.norm(r.double())) * (1 + 1e-5)


def test_standalone_kernel_status_126():
  from aggregathor_b200.ops import gar as gar_ops
  G, r = _case(4, 64, 1, "plain")
  launcher = gar_ops.FusedLauncher(torch.device("cuda"), 4)
  Gc = G.cuda()
  rows = [Gc.data_ptr() + i * 64 * 4 for i in range(4)]
  out = torch.empty(64, device="cuda")
  with pytest.raises(RuntimeError, match="status 126"):   # no root
    launcher.launch(FusedSpec("fltrust", 4), rows, 0, 64, agg_out=out)
  with pytest.raises(RuntimeError, match="status 126"):   # a pre-aggregation bit
    launcher.launch(FusedSpec("fltrust", 4, mix="nnm"), rows, 0, 64, agg_out=out, root=r.cuda(), staging=torch.empty(4, 64, device="cuda"))
  with pytest.raises(RuntimeError, match="status 111"):   # no bucketed phase A
    launcher.phase_a(FusedSpec("fltrust", 4), rows, [(0, 32), (32, 64)], 0, agg_out=out, root=r.cuda())
  torch.cuda.synchronize()


def test_double_and_many_rows_use_the_torch_reference():
  from aggregathor_b200.ops import gar as gar_ops
  G, r = _case(40, 257, 3, "mixed")
  _equal_bits(gar_ops.aggregate(FusedSpec("fltrust", 40), G.cuda(), root=r.cuda()), _ops.torch_fltrust(G.cuda(), r.cuda()))
  out = gar_ops.aggregate(FusedSpec("fltrust", 5), G[:5].double().cuda(), root=r.double().cuda())
  assert out.dtype == torch.float64 and torch.equal(out, _ops.torch_fltrust(G[:5].double().cuda(), r.double().cuda()))


def _manager(engine, opt="sgd", attack=None, k=2, n=8, use_graphs=None, rate=0.05):
  from aggregathor_b200.engine.trainer import Manager
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate("fltrust", n, k, ["root-size:64"])
  return Manager(experiment, gar, n, opt, [], "fixed", ["initial-rate:%g" % rate], device="cuda", engine=engine, seed=7,
                 attack=attacks.instantiate(attack, n, k, []) if attack else None, nb_real_byz=k if attack else 0, use_graphs=use_graphs)


@pytest.mark.parametrize("attack", [None, "alie", "label-flip"])
def test_fused_engine_matches_the_baseline_engine(attack):
  fused = _manager("fused", "sgd", attack)
  base = _manager("baseline", "sgd", attack)
  assert fused.aggregation.name == "fused" and base.aggregation.name == "baseline" and fused.root_ctx is not None
  for _ in range(4):
    fused.train()
    base.train()
    torch.cuda.synchronize()
    _equal_bits(fused.params, base.params)
    _equal_bits(fused.aggregation.root, base.aggregation.root)   # the same parameters, hence the same root gradient
  assert bool(torch.isfinite(fused.params).all())
  fused.close()
  base.close()


@pytest.mark.parametrize("opt", ["sgd", "adam"])
def test_fused_and_baseline_aggregates_agree_under_each_optimizer(opt):
  """The same rows and root on both engines: the aggregated gradients are the same bits at every step; the parameters follow each
  engine's own optimizer update (the fused kernel's, the baseline's SGD kernel or torch update)."""
  from aggregathor_b200.engine.flat import FlatLayout
  from aggregathor_b200.engine.optimizers import optimizers
  from aggregathor_b200.engine.schedules import build
  from aggregathor_b200.parallel.aggregation import BaselineAggregation, FusedAggregation
  layout = FlatLayout()
  layout.add("w", (1000, 37))
  layout.add("b", (37,))
  layout.freeze()
  gar = aggregators.instantiate("fltrust", 8, 2, [])
  fused = FusedAggregation(gar, layout, 8, build(optimizers, "optimizer", opt, []), device="cuda", keep_aggregate=True)
  base = BaselineAggregation(gar, layout, 8, build(optimizers, "optimizer", opt, []), device="cuda")
  gen = torch.Generator().manual_seed(5)
  init = torch.randn(layout.padded_size, generator=gen)
  fused.params.copy_(init)
  base.params.copy_(init)
  for step in range(4):
    r = torch.randn(layout.padded_size, generator=gen) * 0.1
    G = 0.5 * r + torch.randn(8, layout.padded_size, generator=gen) * 0.1
    G[7] = -3.0 * r
    fused.grads.copy_(G)
    base.grads.copy_(G)
    fused.root.copy_(r)
    base.root.copy_(r)
    fused.step(0.05)
    base.step(0.05)
    torch.cuda.synchronize()
    _equal_bits(fused.last_aggregate, base.last_aggregate)
    if opt == "sgd":
      _equal_bits(fused.params, base.params)
    else:
      assert float((fused.params - base.params).abs().max()) <= 1e-4 * max(1.0, float(base.params.abs().max()))


def test_whole_step_graph_replay_matches_eager_steps():
  graphed = _manager("fused", attack="label-flip", use_graphs=True)
  eager = _manager("fused", attack="label-flip", use_graphs=False)
  for _ in range(6):
    a, b = float(graphed.train()), float(eager.train())
    torch.cuda.synchronize()
    _equal_bits(graphed.params, eager.params)
    _equal_bits(graphed.aggregation.root, eager.aggregation.root)
    assert abs(a - b) <= 1e-6 * abs(b)   # the per-worker losses are reduced in no fixed order; the gradients are
  assert graphed._graph is not None and graphed._graph_whole and eager._graph is None
  graphed.close()
  eager.close()


def _gpus():
  return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_gpus() < 2, reason="needs at least 2 GPUs")
def test_fused_matches_baseline_on_all_ranks(tmp_path):
  import json
  nproc = max(r for r in range(1, min(_gpus(), 8) + 1) if 8 % r == 0)
  port = 29700 + os.getpid() % 90
  cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1", "--master-port", str(port),
         str(ROOT / "benchmarks" / "gar_bench.py"), "--gar-dim", "1000003", "--gar-iters", "3", "--gar-rules", "fltrust", "--gar-out", str(tmp_path)]
  proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=900, cwd=str(ROOT))
  out = proc.stdout.decode(errors="replace")
  assert proc.returncode == 0, out[-4000:]
  entry = json.loads((tmp_path / ("gar_bench_%d.json" % nproc)).read_text())["results"]["fltrust"]
  assert entry["replicas_identical"], entry
  assert entry["max_abs_diff_vs_baseline"] < 1e-4, entry

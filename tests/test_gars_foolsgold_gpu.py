"""FoolsGold on the H100: the stand-alone sm_90a kernel over consecutive calls against a float64 oracle of its sums, the exact history
step and the torch reference fed its sums (bit for bit), its status codes, the fused engine against the baseline engine, whole-step
CUDA-graph replays against eager steps, and the multi-rank benchmark check."""

import os
import pathlib
import subprocess
import sys

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
  mu = torch.randn(d, generator=gen)
  G = 0.3 * mu + torch.randn((n, d), generator=gen) * torch.rand((n, 1), generator=gen) * 2
  if kind == "sybil" and n > 3:
    G[n - 3:] = G[n - 1]
  elif kind == "nan-inf" and n > 1:
    G[1, d // 3] = float("nan")
    G[n - 1, 0] = float("inf")
  elif kind == "zero":
    G[::2] = 0.0
  elif kind == "huge":
    G[n // 2] = 1e20
  return G


@pytest.mark.parametrize("d", [1003, 40960])
@pytest.mark.parametrize("kind", ["plain", "sybil", "nan-inf", "zero", "huge"])
@pytest.mark.parametrize("n", list(range(1, 33)))
def test_standalone_kernel(n, kind, d):
  from aggregathor_b200.ops import gar as gar_ops
  spec = FusedSpec("foolsgold", n)
  H = torch.zeros(n, d, device="cuda")
  Href = torch.zeros(n, d, device="cuda")
  for call in range(3):
    G = _case(n, d, 1000 * n + 10 * call + d % 7, kind)
    want = H.cpu() + torch.where(torch.isfinite(G), G, torch.zeros_like(G))
    out, P, N, bad, c = gar_ops.aggregate(spec, G.cuda(), history=H, return_details=True)
    _equal_bits(H, want)
    # the sums of the updated histories against float64, within 1e-5 of ||H_i|| ||H_j||, where fp32 can hold them
    Hd = want.double().numpy()
    norms = np.linalg.norm(Hd, axis=1)
    exact = Hd @ Hd.T
    finite = np.outer(norms, norms) < 1e38
    assert np.all(np.abs(P.astype(np.float64) - exact)[finite] <= (1e-5 * np.outer(norms, norms) + 1e-30)[finite])
    assert np.array_equal(bad, ~torch.isfinite(G).all(dim=1).numpy())
    # given the kernel's sums, the torch reference produces the same history, coefficients and bits
    ref, *details = _ops.torch_foolsgold(G.cuda(), Href, sums=(P, N, bad), return_details=True)
    _equal_bits(Href, H)
    assert np.array_equal(details[3], c)
    _equal_bits(out, ref)
    if kind == "sybil" and n > 3 and c.any():
      assert (c[n - 3:] == 0).all()
    if kind == "nan-inf" and n > 1:
      assert c[1] == 0 and c[n - 1] == 0 and bool(torch.isfinite(out).all())
    if kind == "huge" and n > 1:
      assert c[n // 2] == 0   # its squared norm overflows fp32


def test_status_codes():
  from aggregathor_b200.ops import gar as gar_ops
  n, d = 4, 64
  G = _case(n, d, 1, "plain").cuda()
  launcher = gar_ops.FusedLauncher(torch.device("cuda"), n)
  rows = [G.data_ptr() + i * d * 4 for i in range(n)]
  out = torch.empty(d, device="cuda")
  H = torch.zeros(n, d, device="cuda")
  with pytest.raises(RuntimeError, match="status 127"):   # no history
    launcher.launch(FusedSpec("foolsgold", n), rows, 0, d, agg_out=out)
  for mix in ("nnm", "arc"):   # a pre-aggregation bit
    with pytest.raises(RuntimeError, match="status 128"):
      launcher.launch(FusedSpec("foolsgold", n, f=1, mix=mix), rows, 0, d, agg_out=out, history=H, staging=torch.empty(n, d, device="cuda"))
  with pytest.raises(RuntimeError, match="status 128"):
    launcher.launch(FusedSpec("foolsgold", 2, mix="bucketing", bucket_size=2), rows, 0, d, agg_out=out, history=H,
                    staging=torch.empty(n, d, device="cuda"))
  with pytest.raises(RuntimeError, match="status 129"):   # no bucketed phase A
    launcher.phase_a(FusedSpec("foolsgold", n), rows, [(0, 32), (32, 64)], 0, agg_out=out, history=H)
  with pytest.raises(RuntimeError, match="status 129"):   # nothing pre-accumulated
    launcher.launch(FusedSpec("foolsgold", n), rows, segments=[(0, 32), (32, 64)], agg_out=out, history=H, first_seg=1)
  torch.cuda.synchronize()
  assert not bool(H.any())   # refused launches leave the history alone


def test_double_and_many_rows_use_the_torch_reference():
  from aggregathor_b200.ops import gar as gar_ops
  G = _case(40, 257, 3, "plain").cuda()
  H1, H2 = torch.zeros_like(G), torch.zeros_like(G)
  for _ in range(2):
    _equal_bits(gar_ops.aggregate(FusedSpec("foolsgold", 40), G, history=H1), _ops.torch_foolsgold(G, H2))
    _equal_bits(H1, H2)
  Gd = G[:5].double()
  H1, H2 = torch.zeros_like(Gd), torch.zeros_like(Gd)
  out = gar_ops.aggregate(FusedSpec("foolsgold", 5), Gd, history=H1)
  assert out.dtype == torch.float64 and torch.equal(out, _ops.torch_foolsgold(Gd, H2)) and torch.equal(H1, H2)


def _manager(engine, opt="sgd", attack=None, k=2, n=8, use_graphs=None, rate=0.05):
  from aggregathor_b200.engine.trainer import Manager
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate("foolsgold", n, k, [])
  return Manager(experiment, gar, n, opt, [], "fixed", ["initial-rate:%g" % rate], device="cuda", engine=engine, seed=7,
                 attack=attacks.instantiate(attack, n, k, []) if attack else None, nb_real_byz=k if attack else 0, use_graphs=use_graphs)


@pytest.mark.parametrize("attack", [None, "alie", "label-flip", "backdoor"])
def test_fused_engine_matches_the_baseline_engine(attack):
  fused = _manager("fused", "sgd", attack)
  base = _manager("baseline", "sgd", attack)
  assert fused.aggregation.name == "fused" and base.aggregation.name == "baseline"
  for _ in range(4):
    fused.train()
    base.train()
    torch.cuda.synchronize()
    _equal_bits(fused.params, base.params)
    _equal_bits(fused.aggregation.full_history(), base.aggregation.history)
  assert bool(torch.isfinite(fused.params).all()) and bool(base.aggregation.history.any())
  _equal_bits(fused.state_dict()["aggregation"]["rule_state"], base.aggregation.history)
  fused.close()
  base.close()


def test_fused_and_baseline_aggregates_agree_under_adam():
  """The same rows on both engines: the aggregated gradients and the histories are the same bits at every step."""
  from aggregathor_b200.engine.flat import FlatLayout
  from aggregathor_b200.engine.optimizers import optimizers
  from aggregathor_b200.engine.schedules import build
  from aggregathor_b200.parallel.aggregation import BaselineAggregation, FusedAggregation
  layout = FlatLayout()
  layout.add("w", (1000, 37))
  layout.add("b", (37,))
  layout.freeze()
  gar = aggregators.instantiate("foolsgold", 8, 2, [])
  fused = FusedAggregation(gar, layout, 8, build(optimizers, "optimizer", "adam", []), device="cuda", keep_aggregate=True)
  base = BaselineAggregation(gar, layout, 8, build(optimizers, "optimizer", "adam", []), device="cuda")
  gen = torch.Generator().manual_seed(5)
  init = torch.randn(layout.padded_size, generator=gen)
  fused.params.copy_(init)
  base.params.copy_(init)
  for step in range(4):
    mu = torch.randn(layout.padded_size, generator=gen) * 0.1
    G = 0.5 * mu + torch.randn(8, layout.padded_size, generator=gen) * 0.1
    G[6] = G[7] = -3.0 * mu
    fused.grads.copy_(G)
    base.grads.copy_(G)
    fused.step(0.05)
    base.step(0.05)
    torch.cuda.synchronize()
    _equal_bits(fused.last_aggregate, base.last_aggregate)
    _equal_bits(fused.full_history(), base.history)
    assert float((fused.params - base.params).abs().max()) <= 1e-4 * max(1.0, float(base.params.abs().max()))


def test_whole_step_graph_replay_matches_eager_steps():
  graphed = _manager("fused", attack="label-flip", use_graphs=True)
  eager = _manager("fused", attack="label-flip", use_graphs=False)
  for _ in range(6):
    a, b = float(graphed.train()), float(eager.train())
    torch.cuda.synchronize()
    _equal_bits(graphed.params, eager.params)
    _equal_bits(graphed.aggregation.history, eager.aggregation.history)
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
  port = 29700 + (os.getpid() + 31) % 90
  cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1", "--master-port", str(port),
         str(ROOT / "benchmarks" / "gar_bench.py"), "--gar-dim", "1000003", "--gar-iters", "3", "--gar-rules", "foolsgold", "--gar-out", str(tmp_path)]
  proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=900, cwd=str(ROOT))
  out = proc.stdout.decode(errors="replace")
  assert proc.returncode == 0, out[-4000:]
  entry = json.loads((tmp_path / ("gar_bench_%d.json" % nproc)).read_text())["results"]["foolsgold"]
  assert entry["replicas_identical"], entry
  assert entry["max_abs_diff_vs_baseline"] < 1e-4, entry
  assert entry["history_max_abs_diff_vs_baseline"] == 0.0, entry

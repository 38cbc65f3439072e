"""Mimic on the H100: the sm_90a warm-up and copy kernels against the torch reference, a trajectory through the warm-up and beyond,
several owned segments, the fused and baseline engines bit for bit, a checkpoint round trip, and the exchanges over several GPUs."""

import pytest
import torch

from aggregathor_b200 import aggregators, attacks, experiments
from aggregathor_b200.aggregators import _ops

pytestmark = pytest.mark.gpu


def _rows(gen, n, d, spread, base):
  coef = torch.linspace(-spread, spread, n)[torch.randperm(n, generator=gen)]
  return (coef[:, None] * base[None, :] + 0.05 * torch.randn((n, d), generator=gen)).float()


def _bits(t):
  return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("n,k", [(3, 1), (8, 1), (8, 2), (9, 1), (9, 2), (17, 1), (17, 2), (32, 1), (32, 2)])   # H >= 2
def test_kernel_matches_the_reference(n, k):
  from aggregathor_b200.ops import gar as gar_ops
  d = 40_001   # not a multiple of 4: the op pads the rows and z
  gen = torch.Generator().manual_seed(n * 10 + k)
  base = torch.randn(d, generator=gen)
  byz = list(range(n - k, n))
  honest = [i for i in range(n) if i not in byz]
  ref_state, dev_state = _ops.mimic_state(d), _ops.mimic_state(d, "cuda")
  warmup = 4
  for step in range(6):
    G = _rows(gen, n, d, 1.0 + 0.2 * step, base)
    Gr, Gd = G.clone(), G.cuda()
    ref = _ops.torch_mimic_step_(Gr, byz, ref_state, warmup, return_details=True)
    got = gar_ops.craft_byzantine_(Gd, byz, "mimic", state=dev_state, warmup=warmup, return_details=True)
    torch.cuda.synchronize()
    assert dev_state["t"] == ref_state["t"] == min(step + 1, warmup)
    target = int(dev_state["istar"][0])
    assert target == int(ref_state["istar"][0]) and target in honest
    for b in byz:
      assert torch.equal(_bits(Gd[b].cpu()), _bits(G[target]))
    assert torch.equal(_bits(Gd[honest].cpu()), _bits(G[honest]))
    z, zr = dev_state["z"].cpu().double(), ref_state["z"].double()
    assert float((z - zr).norm()) <= 1e-5 * float(zr.norm())
    if step < warmup:
      s, q, norm2, inv = got
      rs, rq, rnorm2, rinv = ref
      scale = max(abs(v) for v in rs)
      assert all(abs(a - b) <= 1e-4 * scale for a, b in zip(s, rs))
      qscale = max(abs(v) for v in rq)
      assert all(abs(a - b) <= 1e-4 * qscale for a, b in zip(q, rq))
      assert abs(norm2 - rnorm2) <= 1e-4 * rnorm2 and abs(inv - rinv) <= 1e-4 * rinv
    else:
      assert got is None


def test_trajectory_through_the_warmup():
  from aggregathor_b200.ops import gar as gar_ops
  n, k, d, warmup = 10, 2, 100_003, 8
  gen = torch.Generator().manual_seed(3)
  byz = [3, 7]   # not the last slots
  ref_state, dev_state = _ops.mimic_state(d), _ops.mimic_state(d, "cuda")
  targets, ref_targets = [], []
  for step in range(14):
    base = torch.randn(d, generator=gen) if step % 3 == 0 else base
    G = _rows(gen, n, d, 1.0 + 0.3 * (step % 4), base)
    _ops.torch_mimic_step_(G.clone(), byz, ref_state, warmup)
    Gd = G.cuda()
    gar_ops.craft_byzantine_(Gd, byz, "mimic", state=dev_state, warmup=warmup)
    targets.append(int(dev_state["istar"][0]))
    ref_targets.append(int(ref_state["istar"][0]))
    assert torch.equal(_bits(Gd[3].cpu()), _bits(G[targets[-1]])) and torch.equal(_bits(Gd[7].cpu()), _bits(G[targets[-1]]))
  assert targets == ref_targets
  assert len(set(targets[warmup:])) == 1


def _manager(engine, warmup=3, seed=7):
  from aggregathor_b200.engine.trainer import Manager
  n, k = 8, 2
  experiment = experiments.instantiate("mnist", ["batch-size:16", "dirichlet:0.3"])
  gar = aggregators.instantiate("krum", n, k, [])
  return Manager(experiment, gar, n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cuda", engine=engine, seed=seed,
                 attack=attacks.instantiate("mimic", n, k, ["warmup:%d" % warmup]), nb_real_byz=k)


def test_fused_engine_matches_the_baseline_engine():
  fused, base = _manager("fused"), _manager("baseline")
  assert fused.aggregation.name == "fused" and base.aggregation.name == "baseline"
  for step in range(5):
    fused.train()
    base.train()
    torch.cuda.synchronize()
    assert (fused.aggregation.last_craft is None) == (step >= 3)
    assert fused.aggregation.last_craft == base.aggregation.last_craft
    fs, bs = fused.aggregation.attack_state, base.aggregation.attack_state
    assert fs["t"] == bs["t"] and int(fs["istar"][0]) == int(bs["istar"][0])
    assert torch.equal(_bits(fs["z"]), _bits(bs["z"]))
    for i in (6, 7):
      assert torch.equal(_bits(fused.aggregation.visible_rows()[i]), _bits(base.aggregation.visible_rows()[i]))
  assert torch.equal(_bits(fused.params), _bits(base.params))
  fused.close()
  base.close()


def test_checkpoint_resumes_the_trajectory():
  """A restored engine continues the warm-up exactly where the saved one stood: same z, t and i*, then the same updates on the same rows."""
  first = _manager("fused", warmup=4)
  for _ in range(2):
    first.train()
  torch.cuda.synchronize()
  saved = first.state_dict()
  second = _manager("fused", warmup=4, seed=11)
  second.load_state_dict(saved)
  gen = torch.Generator().manual_seed(5)
  d = first.aggregation.d
  base = torch.randn(d, generator=gen)
  for _ in range(3):
    rows = _rows(gen, 8, d, 2.0, base).cuda()
    for mgr in (first, second):
      mgr.aggregation.grads.copy_(rows)
      mgr.aggregation.craft_byzantine([6, 7], "mimic", None, warmup=4)
    torch.cuda.synchronize()
    a, b = first.aggregation.attack_state, second.aggregation.attack_state
    assert a["t"] == b["t"] and int(a["istar"][0]) == int(b["istar"][0])
    assert torch.equal(_bits(a["z"]), _bits(b["z"]))
    assert torch.equal(_bits(first.aggregation.grads), _bits(second.aggregation.grads))
  assert first.aggregation.attack_state["t"] == 4
  first.close()
  second.close()


def test_segments_hold_z_in_owned_order():
  """Several owned segments, out of coordinate order as the fused engine's buckets are: z and y are packed segment after segment; the
  kernel follows the reference (same i*, z within tolerance, Byzantine rows bit-equal to h_{i*})."""
  from aggregathor_b200.ops import gar as gar_ops
  n, k, d, warmup = 9, 2, 60_000, 5
  gen = torch.Generator().manual_seed(9)
  base = torch.randn(d, generator=gen)
  byz = [7, 8]
  honest = list(range(7))
  segments = [(36_000, d), (0, 20_000), (20_000, 36_000)]
  pack = lambda v: torch.cat([v[lo:hi] for lo, hi in segments])
  ref_state = _ops.mimic_state(d)
  state = {"t": 0, "z": pack(_ops.mimic_state(d, "cuda")["z"]), "istar": torch.full((1,), -1, dtype=torch.int32, device="cuda")}
  launcher = gar_ops._launcher(torch.device("cuda", torch.cuda.current_device()), n)
  for step in range(7):
    G = _rows(gen, n, d, 1.0 + 0.2 * step, base)
    _ops.torch_mimic_step_(G.clone(), byz, ref_state, warmup)
    Gd = G.cuda()
    gar_ops.craft([Gd.data_ptr() + i * d * 4 for i in range(n)], segments, honest, byz, "mimic", None, launcher=launcher, state=state, warmup=warmup)
    torch.cuda.synchronize()
    target = int(state["istar"][0])
    assert state["t"] == ref_state["t"] and target == int(ref_state["istar"][0])
    for b in byz:
      assert torch.equal(_bits(Gd[b].cpu()), _bits(G[target]))
    z, zr = state["z"].cpu().double(), pack(ref_state["z"]).double()
    assert float((z - zr).norm()) <= 1e-5 * float(zr.norm())


def _gpus():
  return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_gpus() < 2, reason="needs at least 2 GPUs")
def test_sharded_crafting_on_several_gpus(tmp_path):
  """n = 8 over 2 or 4 ranks, both Byzantine workers on the last rank: the two exchanges give every rank the same i*, and the Byzantine
  rows every rank sees equal the baseline engine's bit for bit."""
  import json
  import os
  import pathlib
  import subprocess
  import sys
  root = pathlib.Path(__file__).resolve().parent.parent
  nproc = 4 if _gpus() >= 4 else 2
  port = 29900 + os.getpid() % 90
  cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr", "127.0.0.1", "--master-port", str(port),
         str(root / "benchmarks" / "gar_bench.py"), "--gar-dim", "1000003", "--gar-iters", "3", "--gar-rules", "average,krum", "--gar-out", str(tmp_path),
         "--gar-attack", "mimic", "--gar-attack-args", "warmup:4"]
  proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, cwd=str(root))
  out = proc.stdout.decode(errors="replace")
  assert proc.returncode == 0, out[-4000:]
  results = json.loads((tmp_path / ("gar_bench_%d.json" % nproc)).read_text())["results"]
  for rule in ("average", "krum"):
    entry = results[rule]
    assert entry["attack"] == "mimic" and entry["replicas_identical"], (rule, entry)
    targets = entry["istar_per_rank"]
    assert len(targets) == nproc and len(set(targets)) == 1 and 0 <= targets[0] < 6, (rule, entry)
    assert targets[0] == entry["baseline_istar"] and entry["rows_match_baseline"], (rule, entry)

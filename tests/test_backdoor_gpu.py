"""The backdoor attack on sm_90a: the preprocessing and image-normalisation kernels with the trigger descriptor against the torch replica,
the softmax cross-entropy kernel against the un-poisoned kernel on labels relabelled on the host, the batched worker pass (honest rows bit
for bit those of a run without the attack, Byzantine rows those of a run on batches poisoned by hand, scale:4 rows exactly 4 x the scale:1
rows), the fast paths the attack keeps (whole-step CUDA graph with the same launches, phase-A overlap), and `backdoor-X-acc`."""

import os
import pathlib
import re
import subprocess
import sys

import pytest
import torch

from aggregathor_b200 import aggregators, attacks, experiments
from aggregathor_b200.engine.trainer import Manager
from aggregathor_b200.models import Context
from aggregathor_b200.ops import nn as nn_ops
from aggregathor_b200.ops.preprocess import Preprocessor

pytestmark = pytest.mark.gpu
ROOT = pathlib.Path(__file__).resolve().parent.parent
U23 = 2.0 ** -23


def _bits(t):
  return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _poisoned_by_hand(n, groups, first, q):
  rows = n // groups
  return [b for b in range(n) if b // rows >= first and b % rows < q]


@pytest.fixture
def native():
  from aggregathor_b200.ops import nn_native
  yield nn_native
  nn_native.set_deterministic(False)


def _images(n, size, channels=3, seed=0):
  return torch.randint(0, 256, (n, size, size, channels), dtype=torch.uint8, generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("mode,size,store,training", [("vgg", 224, 256, True), ("vgg", 224, 256, False), ("inception", 299, 320, True), ("inception", 224, 256, False),
                                                       ("cifarnet", 32, 32, True), ("cifarnet", 32, 32, False), ("plain", 28, 28, False)])
def test_preprocess_kernel_with_the_trigger(mode, size, store, training):
  """Against `Preprocessor._torch` with the same descriptor, to the tolerance of the existing preprocessing test; the images it does not
  poison, and a descriptor that poisons nothing, give the bits of the existing entry point."""
  channels = 1 if mode == "plain" else 3
  x = _images(16, store, channels, seed=3).cuda()
  kwargs = dict(mean=(128.0, 128.0, 128.0), scale=1 / 128.0) if mode == "plain" else {}
  pre = Preprocessor(mode, size, seed=11, **kwargs)
  pre.counter("cuda").fill_(7)
  trigger = (4, 1, 2)
  poisoned = _poisoned_by_hand(16, *trigger)
  for dtype in (torch.float32, torch.bfloat16):
    plain = pre(x, dtype, training, backend="native", advance=False)
    got = pre(x, dtype, training, backend="native", advance=False, trigger=trigger)
    reference = pre._torch(x, torch.float32, training, 7, pre.seed, trigger)
    diff = (got.float() - reference).abs()
    scale = float(reference.abs().max())
    if dtype == torch.float32:
      assert float((diff > 2e-3 * max(scale, 1.0)).float().mean()) < 5e-3, float(diff.max())
    else:
      assert float((diff > 0.01 * max(scale, 1.0) + 1e-2).float().mean()) < 5e-3, float(diff.max())
    clean = [b for b in range(16) if b not in poisoned]
    assert torch.equal(_bits(got[clean]), _bits(plain[clean]))
    assert not torch.equal(got[poisoned], plain[poisoned])
    assert torch.equal(_bits(pre(x, dtype, training, backend="native", advance=False, trigger=(4, 1, 0))), _bits(plain))
  with pytest.raises(ValueError):
    pre(x, torch.float32, training, backend="native", advance=False, trigger=(3, 1, 2))   # 16 images are not 3 groups


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("mode,channels,size", [("vgg", 3, 224), ("inception", 3, 64), ("lenet", 1, 28)])
def test_image_normalize_kernel_with_the_trigger(mode, channels, size, dtype):
  x = _images(12, size, channels, seed=5).cuda()
  trigger = (3, 1, 2)
  got = nn_ops.image_normalize("native", x, mode, dtype, trigger)
  reference = nn_ops.image_normalize("torch", x, mode, dtype, trigger)
  assert float((got.float() - reference.float()).abs().max()) <= 1e-2   # the tolerance of the existing image_normalize test
  plain = nn_ops.image_normalize("native", x, mode, dtype)
  poisoned = _poisoned_by_hand(12, *trigger)
  clean = [b for b in range(12) if b not in poisoned]
  assert torch.equal(_bits(got[clean]), _bits(plain[clean])) and not torch.equal(got[poisoned], plain[poisoned])
  assert torch.equal(_bits(nn_ops.image_normalize("native", x, mode, dtype, (3, 1, 0))), _bits(plain))
  assert torch.equal(_bits(got), _bits(nn_ops.image_normalize("native", nn_ops.stamp_trigger(x, *trigger), mode, dtype)))


def _assert_group_losses(got, ref, rows):
  """A group's loss is a sum of fp32 atomics in an unspecified order: within the reordering bound of `rows` non-negative addends."""
  assert bool(((got - ref).abs() <= 2 * rows * U23 * ref.abs()).all()), (got, ref)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("smoothing", [0.0, 0.1])
@pytest.mark.parametrize("groups", [1, 4, 8])
@pytest.mark.parametrize("k", [10, 1001])
def test_xent_kernel_relabels_and_scales(native, k, groups, smoothing, dtype):
  rows, target, q = 5, 7, 3
  b = rows * groups
  gen = torch.Generator().manual_seed(k + groups)
  ld = k + 8 - k % 8
  logits = (torch.randn((b, ld), generator=gen) * 6).to(dtype).cuda()[:, :k]   # strided rows
  labels = torch.randint(0, k, (b,), generator=gen).cuda()
  for first in range(groups + 1):
    relabelled = labels.cpu().clone()
    for r in _poisoned_by_hand(b, groups, first, q):
      relabelled[r] = target
    ref_loss, ref_d = native.softmax_xent(logits, relabelled.cuda(), smoothing, groups)
    loss1, d1 = native.softmax_xent(logits, labels, smoothing, groups, backdoor=(first, q, target, 1.0))
    loss4, d4 = native.softmax_xent(logits, labels, smoothing, groups, backdoor=(first, q, target, 4.0))
    torch.cuda.synchronize()
    assert torch.equal(_bits(d1), _bits(ref_d)), first
    lo = first * rows
    assert torch.equal(_bits(d4[:lo]), _bits(d1[:lo])) and torch.equal(_bits(d4[lo:]), _bits(d1[lo:] * 4)), first
    _assert_group_losses(loss1, ref_loss, rows)
    _assert_group_losses(loss4, ref_loss, rows)   # the loss is not scaled
  for bad in ((groups + 1, q, target, 1.0), (0, rows + 1, target, 1.0), (0, q, k, 1.0), (0, q, target, 0.0), (0, q, target, float("nan"))):
    with pytest.raises(RuntimeError, match="status 303"):
      native.softmax_xent(logits, labels, smoothing, groups, backdoor=bad)


class _PoisonedStream:
  """A Byzantine worker's stream poisoned on the host: the first q samples relabelled to the target and, with `stamp`, stamped."""

  def __init__(self, stream, q, target, stamp):
    self.stream, self.q, self.target, self.stamp = stream, q, target, stamp

  def __iter__(self):
    return self

  def __next__(self):
    x, y = next(self.stream)
    y = y.clone()
    y[:self.q] = self.target
    return (nn_ops.stamp_trigger(x, 1, 0, self.q) if self.stamp else x), y


_BATCHED = {"cnnet": ("cnnet", ["batch-size:8"]),
            "resnet": ("slim-resnet_v1_50-imagenet", ["batch-size:2", "image-size:64", "synthetic-samples:64"])}


@pytest.mark.parametrize("name", sorted(_BATCHED))
def test_batched_pass_rows(native, name):
  """One rank, w = 4 workers in one batched pass, the last 2 Byzantine: honest rows and batch-norm statistics are those of the run without
  the attack; Byzantine rows are those of a run on batches poisoned by hand (ResNet-50 on synthetic data, normalised by
  `image_normalize`: stamped and relabelled on the host; cnnet, whose trigger follows the random crop: relabelled on the host and stamped
  by the preprocessing kernel); the rows at scale:4 are exactly 4 x those at scale:1."""
  native.set_deterministic(True)   # weight gradients in one accumulation chain: bit-reproducible rows
  n, k, target = 4, 2, 1
  experiment, args = _BATCHED[name]
  q = int(args[0].split(":")[1]) // 2

  def manager(attack_args=None):
    gar = aggregators.instantiate("average", n, 0, [])
    attack = attacks.instantiate("backdoor", n, k, attack_args) if attack_args is not None else None
    return Manager(experiments.instantiate(experiment, list(args)), gar, n, "sgd", [], "fixed", ["initial-rate:0.01"], device="cuda",
                   attack=attack, nb_real_byz=k if attack is not None else 0, seed=5)

  bd, bd4, plain, by_hand = manager(["target:%d" % target]), manager(["target:%d" % target, "scale:4"]), manager(), manager()
  stamp = name == "resnet"
  by_hand.streams = [_PoisonedStream(s, q, target, stamp) if i >= n - k else s for i, s in zip(by_hand.local_workers, by_hand.streams)]
  if not stamp:
    by_hand.experiment.trigger = lambda ctx: (ctx.groups, n - k, q) if ctx.groups > 1 else None
  assert bd.batched and plain.batched and by_hand.batched
  assert bd.batched_ctx.backdoor == (n - k, q, target, 1.0) and plain.batched_ctx.backdoor is None and bd.eval_ctx.backdoor is None
  losses = {}
  for tag, mgr in (("bd", bd), ("bd4", bd4), ("plain", plain), ("by_hand", by_hand)):
    losses[tag] = torch.stack([l.float() for l in mgr.compute_gradients()])
    torch.cuda.synchronize()
  assert bool(torch.isfinite(bd.grads).all())
  for i in range(n):
    ref = by_hand if i >= n - k else plain
    assert torch.equal(_bits(bd.grads[i]), _bits(ref.grads[i])), i
  for i in range(n):   # every layer's backward is linear in dy: a power of two scales it exactly
    assert torch.equal(_bits(bd4.grads[i]), _bits(bd.grads[i] * (4 if i >= n - k else 1))), i
  assert not torch.equal(bd.grads[n - 1], plain.grads[n - 1])
  torch.testing.assert_close(losses["bd"][:n - k], losses["plain"][:n - k], rtol=1e-5, atol=0)   # fp32 atomics in varying order
  torch.testing.assert_close(losses["bd"][n - k:], losses["by_hand"][n - k:], rtol=1e-5, atol=0)
  torch.testing.assert_close(losses["bd4"], losses["bd"], rtol=1e-5, atol=0)
  for key, value in bd.states.items():
    assert torch.equal(_bits(value), _bits(plain.states[key])), key
  for mgr in (bd, bd4, plain, by_hand):
    mgr.close()


def _fused(experiment, exp_args, attack, **kwargs):
  n = 8
  gar = aggregators.instantiate("krum", n, 2, [])
  return Manager(experiments.instantiate(experiment, list(exp_args)), gar, n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cuda", engine="fused", seed=3,
                 attack=attacks.instantiate("backdoor", n, 2, ["scale:2"]) if attack else None, nb_real_byz=2 if attack else 0, **kwargs)


@pytest.mark.parametrize("experiment,exp_args", [("mnist", ["batch-size:16"]), ("cnnet", ["batch-size:16", "eval-batch-size:256"])])
def test_whole_step_graph_is_kept(native, monkeypatch, experiment, exp_args):
  """The backdoor run captures the whole step (workers + aggregation) with exactly the launches of the run without the attack, and its
  replayed steps equal an eager run of the same attack."""
  native.set_deterministic(True)
  bd, plain = _fused(experiment, exp_args, True), _fused(experiment, exp_args, False)
  for _ in range(5):
    bd.train()
    plain.train()
  torch.cuda.synchronize()
  assert bd._graph is not None and bd._graph_whole and plain._graph is not None and plain._graph_whole
  assert bd._graph_launches == plain._graph_launches > 0
  assert not torch.equal(bd.params, plain.params)
  monkeypatch.setenv("AGB_NO_GRAPH", "1")
  eager = _fused(experiment, exp_args, True)
  for _ in range(5):
    eager.train()
  torch.cuda.synchronize()
  assert eager._graph is None
  assert torch.equal(_bits(bd.params), _bits(eager.params))
  for mgr in (bd, plain, eager):
    mgr.close()


def test_phase_a_overlap_is_kept(monkeypatch):
  monkeypatch.setenv("AGB_OVERLAP", "2")
  bd, plain = _fused("cnnet", ["batch-size:16"], True), _fused("cnnet", ["batch-size:16"], False)
  assert plain._bucket_layers and len(bd._bucket_layers) == len(plain._bucket_layers)
  assert len(bd.aggregation.buckets) == len(plain.aggregation.buckets) > 1
  for _ in range(4):
    bd.train()
  torch.cuda.synchronize()
  assert bd._graph is not None and bd._graph_whole and bool(torch.isfinite(bd.params).all())
  bd.close()
  plain.close()


@pytest.mark.parametrize("experiment,exp_args", [("mnist", ["batch-size:16"]), ("cnnet", ["batch-size:16", "eval-batch-size:256"])])
def test_evaluate_matches_torch(experiment, exp_args):
  """`backdoor-X-acc` on the GPU: bit for bit the native evaluation of the set stamped on the host, and within 2 % of the fp32 torch
  computation on the same parameters (bf16 logits may flip a near tie)."""
  mgr = _fused(experiment, exp_args, True)
  for _ in range(6):
    mgr.train()
  metrics = mgr.evaluate()
  assert sorted(metrics) == ["backdoor-X-acc", "top1-X-acc"]
  inputs, labels = mgr._backdoor_batch
  assert bool((labels != 0).all())
  stamped = nn_ops.stamp_trigger(inputs, 1, 0, len(labels)).cuda()
  exp = mgr.experiment
  with torch.no_grad():
    logits = mgr.model.logits(exp.preprocess(stamped, mgr.eval_ctx, False), mgr.eval_ctx)
    assert metrics["backdoor-X-acc"] == float((logits.float().argmax(dim=1) == 0).float().mean())
    ctx = Context("torch", False, torch.float32, "cuda")
    ctx.weights, ctx.master, ctx.state = mgr.master_views, mgr.master_views, mgr.states
    logits = mgr.model.logits(exp.preprocess(stamped, ctx, False), ctx)
  assert abs(metrics["backdoor-X-acc"] - float((logits.argmax(dim=1) == 0).float().mean())) <= 0.02
  mgr.close()


def _gpus():
  return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_gpus() < 2, reason="needs at least 2 GPUs")
def test_multi_rank_training_keeps_replicas_identical(tmp_path):
  """2 ranks x 4 workers, Krum on cnnet with the overlapped distance pass, the last 2 workers (on rank 1) running the scaled backdoor."""
  workers = '"127.0.0.1:7001", "127.0.0.1:7002"'
  evaluation = tmp_path / "eval"
  args = [str(ROOT / "runner.py"), "--server", '{"ps": ["127.0.0.1:7000"], "workers": [%s], "eval": ["127.0.0.1:7000"]}' % workers, "--no-wait",
          "--experiment", "cnnet", "--experiment-args", "batch-size:16", "--aggregator", "krum", "--nb-workers", "8", "--nb-decl-byz-workers", "2",
          "--nb-real-byz-workers", "2", "--attack", "backdoor", "--attack-args", "target:0", "scale:8", "--max-step", "10", "--use-gpu", "--reuse-gpu",
          "--debug-checksum", "--learning-rate-args", "initial-rate:0.02", "--evaluation-file", str(evaluation), "--checkpoint-dir", str(tmp_path / "c"),
          "--checkpoint-delta", "-1", "--checkpoint-period", "-1", "--summary-dir", "-"]
  port = 29700 + os.getpid() % 200
  cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", str(port)] + args
  proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, cwd=str(ROOT), env=dict(os.environ, AGB_OVERLAP="2"))
  out = proc.stdout.decode(errors="replace")
  assert proc.returncode == 0, out[-4000:]
  assert "Replica divergence" not in out and "Step 9: total loss" in out
  assert "forward/backward + aggregation into a CUDA graph" in out
  losses = [float(x) for x in re.findall(r"Step \d+: total loss = ([0-9.eE+-]+)", out)]
  assert len(losses) == 10 and all(l == l for l in losses)
  assert "backdoor-X-acc:" in evaluation.read_text()

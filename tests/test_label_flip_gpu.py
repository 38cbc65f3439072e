"""The label-flipping attack on sm_90a: the softmax cross-entropy kernel with `flip_from` against the unflipped kernel on labels flipped
on the host, the batched worker pass (honest rows bit for bit those of a run without the attack, Byzantine rows those of a run on the
flipped labels), and the fast paths the attack keeps: the whole-step CUDA graph with the same launches, and the phase-A overlap."""

import os
import pathlib
import re
import subprocess
import sys

import pytest
import torch

from aggregathor_b200 import aggregators, attacks, experiments
from aggregathor_b200.engine.trainer import Manager

pytestmark = pytest.mark.gpu
ROOT = pathlib.Path(__file__).resolve().parent.parent
U23 = 2.0 ** -23


def _bits(t):
  return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _flipped_by_hand(labels, classes, groups, flip_from):
  host = labels.cpu().clone()
  rows = host.shape[0] // groups
  for r in range(host.shape[0]):
    if r // rows >= flip_from and 0 <= int(host[r]) < classes:
      host[r] = classes - 1 - int(host[r])
  return host.to(labels.device)


@pytest.fixture
def native():
  from aggregathor_b200.ops import nn_native
  yield nn_native
  nn_native.set_deterministic(False)


def _assert_group_losses(got, ref, rows, replicated):
  """A group's loss is a sum of fp32 atomics in an unspecified order: bit-equal when the group's rows are identical (every order adds the
  same addends alike), otherwise within the reordering bound of `rows` non-negative addends."""
  if replicated:
    assert torch.equal(_bits(got), _bits(ref)), (got, ref)
  else:
    assert bool(((got - ref).abs() <= 2 * rows * U23 * ref.abs()).all()), (got, ref)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("smoothing", [0.0, 0.1])
@pytest.mark.parametrize("groups", [1, 4, 8])
@pytest.mark.parametrize("k", [10, 1001])
@pytest.mark.parametrize("replicated", [False, True])
def test_kernel_equals_the_unflipped_kernel_on_flipped_labels(native, replicated, k, groups, smoothing, dtype):
  rows = 5
  b = rows * groups
  gen = torch.Generator().manual_seed(k + groups)
  ld = k + 8 - k % 8
  base = torch.randn((b, ld), generator=gen) * 6
  labels = torch.randint(0, k, (b,), generator=gen)
  labels[0], labels[1], labels[rows - 1] = 0, k - 1, -1
  labels[-1], labels[-2] = k, k + 3   # outside [0, K): never flipped, match no class
  if replicated:
    base = base[::rows].repeat_interleave(rows, dim=0)
    labels = labels[::rows].repeat_interleave(rows)
  logits = base.to(dtype).cuda()[:, :k]   # strided rows
  labels = labels.cuda()
  plain = native.softmax_xent(logits, labels, smoothing, groups)
  for flip_from in range(groups + 1):
    loss, d = native.softmax_xent(logits, labels, smoothing, groups, flip_from)
    ref_loss, ref_d = native.softmax_xent(logits, _flipped_by_hand(labels, k, groups, flip_from), smoothing, groups)
    torch.cuda.synchronize()
    assert torch.equal(_bits(d), _bits(ref_d)), flip_from
    _assert_group_losses(loss, ref_loss, rows, replicated)
    if flip_from < groups:
      assert not torch.equal(d[rows * flip_from:], plain[1][rows * flip_from:])
  # flip_from = groups flips nothing: the existing entry point, bit for bit
  loss, d = native.softmax_xent(logits, labels, smoothing, groups, groups)
  assert torch.equal(_bits(d), _bits(plain[1]))
  _assert_group_losses(loss, plain[0], rows, replicated)
  for bad in (-1, groups + 1):
    with pytest.raises(RuntimeError, match="status 301"):
      native.softmax_xent(logits, labels, smoothing, groups, bad)


def test_native_disabled_fallback_flips_too(monkeypatch):
  from aggregathor_b200.ops import nn as nn_ops, nn_native
  monkeypatch.setattr(nn_native, "_DISABLED", {"xent"})
  monkeypatch.setattr(nn_ops, "_STRICT", False)
  gen = torch.Generator().manual_seed(3)
  logits = (torch.randn((12, 10), generator=gen) * 3).cuda()
  labels = torch.randint(0, 10, (12,), generator=gen).cuda()
  loss, d = nn_ops.softmax_xent("native", logits, labels, 0.1, 4, flip_from=1)
  ref_loss, ref_d = nn_ops.softmax_xent("torch", logits, _flipped_by_hand(labels, 10, 4, 1), 0.1, 4)
  assert torch.equal(loss, ref_loss) and torch.equal(d, ref_d)


class _FlippedStream:
  """A worker's batch stream with its labels flipped on the host (K - 1 - y)."""

  def __init__(self, stream, classes):
    self.stream, self.classes = stream, classes

  def __iter__(self):
    return self

  def __next__(self):
    x, y = next(self.stream)
    return x, _flipped_by_hand(y, self.classes, 1, 0)


_BATCHED = {"cnnet": ("cnnet", ["batch-size:8"]),
            "resnet": ("slim-resnet_v1_50-imagenet", ["batch-size:2", "image-size:64", "synthetic-samples:64"])}


@pytest.mark.parametrize("name", sorted(_BATCHED))
def test_batched_pass_rows(native, name):
  """One rank, w = 4 workers in one batched pass, the last 2 Byzantine: honest rows (and the batch-norm statistics) are those of the run
  without the attack, Byzantine rows those of the run without the attack on the flipped labels, bit for bit."""
  native.set_deterministic(True)   # weight gradients in one accumulation chain: bit-reproducible rows
  n, k = 4, 2
  experiment, args = _BATCHED[name]

  def manager(attack=None):
    gar = aggregators.instantiate("average", n, 0, [])
    return Manager(experiments.instantiate(experiment, list(args)), gar, n, "sgd", [], "fixed", ["initial-rate:0.01"], device="cuda",
                   attack=attack, nb_real_byz=k if attack is not None else 0, seed=5)

  lf, plain, by_hand = manager(attacks.instantiate("label-flip", n, k, [])), manager(), manager()
  classes = lf.model.num_classes
  by_hand.streams = [_FlippedStream(s, classes) if i >= n - k else s for i, s in zip(by_hand.local_workers, by_hand.streams)]
  assert lf.batched and plain.batched and by_hand.batched
  assert lf.batched_ctx.flip_from == n - k and plain.batched_ctx.flip_from is None and lf.eval_ctx.flip_from is None
  losses = {}
  for tag, mgr in (("lf", lf), ("plain", plain), ("by_hand", by_hand)):
    losses[tag] = torch.stack([l.float() for l in mgr.compute_gradients()])
    torch.cuda.synchronize()
  assert bool(torch.isfinite(lf.grads).all())
  for i in range(n):
    ref = by_hand if i >= n - k else plain
    assert torch.equal(_bits(lf.grads[i]), _bits(ref.grads[i])), i
  assert not torch.equal(lf.grads[n - 1], plain.grads[n - 1])
  torch.testing.assert_close(losses["lf"][:n - k], losses["plain"][:n - k], rtol=1e-5, atol=0)   # fp32 atomics in varying order
  torch.testing.assert_close(losses["lf"][n - k:], losses["by_hand"][n - k:], rtol=1e-5, atol=0)
  for key, value in lf.states.items():
    assert torch.equal(_bits(value), _bits(plain.states[key])), key
  for mgr in (lf, plain, by_hand):
    mgr.close()


def _fused(attack, **kwargs):
  n = 8
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate("krum", n, 2, [])
  return Manager(experiment, gar, n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cuda", engine="fused", seed=3,
                 attack=attacks.instantiate("label-flip", n, 2, []) if attack else None, nb_real_byz=2 if attack else 0, **kwargs)


def test_whole_step_graph_is_kept(native, monkeypatch):
  """Default graph settings: the label-flipping run captures the whole step (workers + aggregation) with exactly the launches of the run
  without the attack, and its replayed steps equal an eager run of the same attack."""
  native.set_deterministic(True)
  lf, plain = _fused(True), _fused(False)
  for _ in range(5):
    lf.train()
    plain.train()
  torch.cuda.synchronize()
  assert lf._graph is not None and lf._graph_whole and plain._graph is not None and plain._graph_whole
  assert lf._graph_launches == plain._graph_launches > 0
  assert not torch.equal(lf.params, plain.params)
  monkeypatch.setenv("AGB_NO_GRAPH", "1")
  eager = _fused(True)
  for _ in range(5):
    eager.train()
  torch.cuda.synchronize()
  assert eager._graph is None
  assert torch.equal(_bits(lf.params), _bits(eager.params))
  for mgr in (lf, plain, eager):
    mgr.close()


def test_phase_a_overlap_is_kept(monkeypatch):
  monkeypatch.setenv("AGB_OVERLAP", "2")
  n = 8

  def manager(attack):
    experiment = experiments.instantiate("cnnet", ["batch-size:16"])
    gar = aggregators.instantiate("krum", n, 2, [])
    return Manager(experiment, gar, n, "sgd", [], "fixed", ["initial-rate:0.02"], device="cuda", engine="fused",
                   attack=attacks.instantiate("label-flip", n, 2, []) if attack else None, nb_real_byz=2 if attack else 0)

  lf, plain = manager(True), manager(False)
  assert plain._bucket_layers and len(lf._bucket_layers) == len(plain._bucket_layers)
  assert len(lf.aggregation.buckets) == len(plain.aggregation.buckets) > 1
  for _ in range(4):
    lf.train()
  torch.cuda.synchronize()
  assert lf._graph is not None and lf._graph_whole and bool(torch.isfinite(lf.params).all())
  lf.close()
  plain.close()


def _gpus():
  return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.skipif(_gpus() < 2, reason="needs at least 2 GPUs")
def test_multi_rank_training_keeps_replicas_identical(tmp_path):
  """2 ranks x 4 workers, Krum on cnnet with the overlapped distance pass, the last 2 workers flipping their labels (all on rank 1)."""
  workers = '"127.0.0.1:7001", "127.0.0.1:7002"'
  args = [str(ROOT / "runner.py"), "--server", '{"ps": ["127.0.0.1:7000"], "workers": [%s], "eval": ["127.0.0.1:7000"]}' % workers, "--no-wait",
          "--experiment", "cnnet", "--experiment-args", "batch-size:16", "--aggregator", "krum", "--nb-workers", "8", "--nb-decl-byz-workers", "2",
          "--nb-real-byz-workers", "2", "--attack", "label-flip", "--max-step", "10", "--use-gpu", "--reuse-gpu", "--debug-checksum",
          "--learning-rate-args", "initial-rate:0.02", "--evaluation-file", "-", "--checkpoint-dir", str(tmp_path / "c"), "--checkpoint-delta", "-1",
          "--checkpoint-period", "-1", "--summary-dir", "-"]
  port = 29700 + os.getpid() % 200
  cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", str(port)] + args
  proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, cwd=str(ROOT), env=dict(os.environ, AGB_OVERLAP="2"))
  out = proc.stdout.decode(errors="replace")
  assert proc.returncode == 0, out[-4000:]
  assert "Replica divergence" not in out and "Step 9: total loss" in out
  assert "forward/backward + aggregation into a CUDA graph" in out
  losses = [float(x) for x in re.findall(r"Step \d+: total loss = ([0-9.eE+-]+)", out)]
  assert len(losses) == 10 and all(l == l for l in losses)

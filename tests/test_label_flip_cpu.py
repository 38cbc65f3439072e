"""The label-flipping attack (Fang et al., USENIX Security 2020) on the CPU: the torch softmax cross-entropy with `flip_from` against the
same call on labels flipped by hand, the attack's argument checks, a `Manager` whose Byzantine rows are the gradients of the flipped
batches while the honest rows stay bit for bit those of a run without the attack, and the runner CLI."""

import math
import os
import pathlib
import re
import subprocess
import sys

import pytest
import torch

from aggregathor_b200 import aggregators, attacks, experiments, tools
from aggregathor_b200.engine.trainer import Manager
from aggregathor_b200.ops import nn as nn_ops

ROOT = pathlib.Path(__file__).resolve().parent.parent
LOCAL = ["--server", '{"local": ["127.0.0.1:7000"]}', "--ps-job-name", "local", "--wk-job-name", "local", "--ev-job-name", "local", "--no-wait"]


def _flipped_by_hand(labels, classes, groups, flip_from):
  out = labels.clone()
  rows = labels.shape[0] // groups
  for r in range(labels.shape[0]):
    if r // rows >= flip_from and 0 <= int(labels[r]) < classes:
      out[r] = classes - 1 - int(labels[r])
  return out


def _bits(t):
  return t.contiguous().view(torch.int64 if t.dtype == torch.float64 else torch.int32)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("smoothing", [0.0, 0.1])
@pytest.mark.parametrize("groups", [1, 4])
def test_torch_xent_flips_the_groups_from_flip_from(groups, smoothing, dtype):
  classes, rows = 10, 6
  gen = torch.Generator().manual_seed(groups * 10 + int(smoothing * 10))
  logits = (torch.randn((groups * rows, classes), generator=gen) * 4).to(dtype)
  labels = torch.randint(0, classes, (groups * rows,), generator=gen)
  labels[0], labels[-1], labels[rows // 2] = -1, classes, classes + 7   # outside [0, K): left as they are, match no class
  labels[1], labels[-2] = 0, classes - 1
  plain_loss, plain_d = nn_ops.softmax_xent("torch", logits, labels, smoothing, groups)
  for flip_from in range(groups + 1):
    loss, d = nn_ops.softmax_xent("torch", logits, labels, smoothing, groups, flip_from=flip_from)
    ref_loss, ref_d = nn_ops.softmax_xent("torch", logits, _flipped_by_hand(labels, classes, groups, flip_from), smoothing, groups)
    assert loss.dtype == ref_loss.dtype == (torch.float64 if dtype == torch.float64 else torch.float32)
    assert torch.equal(_bits(loss), _bits(ref_loss)) and torch.equal(_bits(d), _bits(ref_d)), flip_from
    flipped = slice(rows * flip_from, None)
    assert torch.equal(_bits(d[:rows * flip_from]), _bits(plain_d[:rows * flip_from]))   # the groups before flip_from are untouched
    if flip_from < groups:
      assert not torch.equal(d[flipped], plain_d[flipped])
  assert torch.equal(_bits(nn_ops.softmax_xent("torch", logits, labels, smoothing, groups, flip_from=None)[1]), _bits(plain_d))


def test_label_outside_the_classes_matches_none():
  logits = torch.tensor([[1.0, 2.0, 3.0], [0.5, -1.0, 2.0]])
  for label in (-1, 3, 17):
    labels = torch.tensor([label, label])
    loss, d = nn_ops.softmax_xent("torch", logits, labels, 0.0, 1, flip_from=0)
    assert float(loss) == 0.0
    torch.testing.assert_close(d, torch.softmax(logits, dim=1) / 2)
  loss, d = nn_ops.softmax_xent("torch", logits, torch.tensor([0, 2]), 0.0, 1, flip_from=0)   # 0 -> 2, 2 -> 0
  ref_loss, ref_d = nn_ops.softmax_xent("torch", logits, torch.tensor([2, 0]), 0.0)
  assert torch.equal(loss, ref_loss) and torch.equal(d, ref_d)


def test_flip_labels_helper():
  labels = torch.tensor([0, 1, 9, 10, -1, 3, 5, 9])
  assert nn_ops.flip_labels(labels, 10, 2, 1).tolist() == [0, 1, 9, 10, -1, 6, 4, 0]
  assert nn_ops.flip_labels(labels, 10, 2, 2).tolist() == labels.tolist()
  assert nn_ops.flip_labels(labels, 10).tolist() == [9, 8, 0, 10, -1, 6, 4, 0]
  for bad in (-1, 3):
    with pytest.raises(ValueError):
      nn_ops.flip_labels(labels, 10, 2, bad)


def test_auxiliary_head_trains_on_the_flipped_labels_too():
  """A batched pass of 3 groups through a model with an auxiliary head, `ctx.flip_from` = 1: the same losses and gradient rows as the
  unflipped pass on labels flipped by hand, so both heads see the flipped labels."""
  from aggregathor_b200.engine.flat import FlatLayout
  from aggregathor_b200.models import Context
  from aggregathor_b200.models.core import AuxHead, Dense, Model, Sequential
  classes, groups, rows = 5, 3, 4
  model = Model("aux", Sequential("aux", [Dense("d1", 12, 16, relu=True), AuxHead("aux", Dense("aux_logits", 16, classes), 0.4),
                                          Dense("logits", 16, classes)]), (12,), classes)
  layout, states = FlatLayout(), {}
  model.declare(layout, states)
  layout.freeze()
  params = torch.zeros(layout.padded_size)
  model.initialize(layout.views(params), {}, torch.Generator().manual_seed(2))
  gen = torch.Generator().manual_seed(4)
  x = torch.randn((groups * rows, 12), generator=gen)
  labels = torch.randint(0, classes, (groups * rows,), generator=gen)

  def run(labels, flip_from):
    ctx = Context("torch", True, torch.float32, "cpu")
    ctx.master = ctx.weights = layout.views(params)
    ctx.state = {}
    grads = torch.zeros((groups, layout.padded_size))
    ctx.grads, ctx.groups, ctx.group_stride, ctx.flip_from = layout.views(grads[0]), groups, grads.stride(0), flip_from
    return model.loss_and_backward(x, labels, ctx), grads

  loss, grads = run(labels, 1)
  ref_loss, ref_grads = run(_flipped_by_hand(labels, classes, groups, 1), None)
  plain_loss, plain_grads = run(labels, None)
  assert torch.equal(_bits(loss), _bits(ref_loss)) and torch.equal(_bits(grads), _bits(ref_grads))
  assert torch.equal(_bits(grads[0]), _bits(plain_grads[0])) and not torch.equal(grads[1:], plain_grads[1:])
  lo, hi = layout.offset("aux_logits/weights"), layout.offset("aux_logits/biases")
  assert not torch.equal(grads[1:, lo:hi], plain_grads[1:, lo:hi])   # the auxiliary head's own gradients changed


def test_registry_and_arguments():
  assert "label-flip" in attacks.itemize()
  attack = attacks.instantiate("label-flip", 5, 2, [])
  assert attack.flips_labels and not attack.omniscient and not attack.forges
  assert attacks.instantiate("label-flip", 5, 5, None).flips_labels   # every worker may flip
  with pytest.raises(tools.UserException, match="takes no argument.*'factor:2'"):
    attacks.instantiate("label-flip", 5, 2, ["factor:2"])
  for k in (0, 6, -1):
    with pytest.raises(tools.UserException, match="between 1 and n"):
      attacks.instantiate("label-flip", 5, k, [])


class _FlippedStream:
  """A worker's batch stream with its labels flipped by hand (K - 1 - y)."""

  def __init__(self, stream, classes):
    self.stream, self.classes = stream, classes

  def __iter__(self):
    return self

  def __next__(self):
    x, y = next(self.stream)
    return x, _flipped_by_hand(y, self.classes, 1, 0)


def _manager(attack=None, k=0, n=5):
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate("average", n, 0, [])
  return Manager(experiment, gar, n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu", backend="torch", attack=attack, nb_real_byz=k, seed=7)


def test_manager_byzantine_rows_are_the_gradients_of_flipped_labels():
  n, k = 5, 2
  lf = _manager(attacks.instantiate("label-flip", n, k, []), k)
  plain = _manager()
  by_hand = _manager()
  by_hand.streams = [_FlippedStream(s, 10) if i >= n - k else s for i, s in zip(by_hand.local_workers, by_hand.streams)]
  assert [ctx.flip_from for ctx in lf.contexts] == [None, None, None, 0, 0] and lf.eval_ctx.flip_from is None
  assert all(ctx.flip_from is None for ctx in plain.contexts)
  losses = {name: [float(l) for l in mgr.compute_gradients()] for name, mgr in (("lf", lf), ("plain", plain), ("by_hand", by_hand))}
  for i in range(n):
    row = lf.grads[lf.placement[i][1]]
    ref, ref_loss = (by_hand, losses["by_hand"][i]) if i >= n - k else (plain, losses["plain"][i])
    assert torch.equal(_bits(row), _bits(ref.grads[ref.placement[i][1]])), i
    assert losses["lf"][i] == ref_loss, i
  for i in range(n - k, n):
    assert not torch.equal(lf.grads[i], plain.grads[i])
  total = float(lf.train())   # the reported total loss sums every worker's, the Byzantine workers' on their flipped labels
  assert math.isfinite(total)
  for mgr in (lf, plain, by_hand):
    mgr.close()


def _run(args, timeout=300):
  env = dict(os.environ, AGB_NUM_THREADS="2", OMP_NUM_THREADS="2")
  proc = subprocess.run([sys.executable, str(ROOT / "runner.py")] + args, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=timeout, env=env, cwd=str(ROOT))
  return proc.returncode, proc.stdout.decode(errors="replace")


def test_runner_label_flip_krum(tmp_path):
  evaluation = tmp_path / "eval"
  args = LOCAL + ["--experiment", "mnist", "--experiment-args", "batch-size:16", "--aggregator", "krum", "--nb-workers", "7", "--nb-decl-byz-workers", "2",
                  "--nb-real-byz-workers", "2", "--attack", "label-flip", "--max-step", "6", "--seed", "3", "--learning-rate-args", "initial-rate:0.05",
                  "--evaluation-file", str(evaluation), "--summary-dir", "-", "--evaluation-delta", "1000", "--evaluation-period", "-1",
                  "--checkpoint-period", "-1", "--checkpoint-delta", "1000"]
  code, out = _run(args)
  assert code == 0, out
  assert "label-flip" in out, out
  losses = [float(x) for x in re.findall(r"Step \d+: total loss = ([0-9.eE+-]+|NaN)", out)]
  assert len(losses) == 6 and all(math.isfinite(x) for x in losses), out
  lines = evaluation.read_text().strip().splitlines()
  assert len(lines) == 2, out   # before training and at the end
  wall, step, metric = lines[-1].split("\t")
  assert int(step) == 6 and float(wall) > 0 and re.fullmatch(r"top1-X-acc:[0-9.eE+-]+", metric), lines
  code, out = _run(args + ["--attack-args", "factor:2"])
  assert code != 0 and "label-flip takes no argument" in out and "factor:2" in out

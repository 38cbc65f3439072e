"""The backdoor attack (BadNets trigger, target label, update scaling) on the CPU: the trigger helper against a hand-written pattern,
the torch preprocessing replica in every mode, the torch softmax cross-entropy, the attack's refusals, torch-backend `Manager`s whose
honest rows are those of a run without the attack and whose Byzantine rows are those of a run on batches poisoned by hand, the
`backdoor-X-acc` metric, FLTrust's root row, the runner's evaluation and event files, and the attack's efficacy on MNIST."""

import math
import os
import pathlib
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from aggregathor_b200 import aggregators, attacks, experiments, tools
from aggregathor_b200.engine.trainer import Manager
from aggregathor_b200.models import Context
from aggregathor_b200.ops import nn as nn_ops
from aggregathor_b200.ops.preprocess import Preprocessor

ROOT = pathlib.Path(__file__).resolve().parent.parent
LOCAL = ["--server", '{"local": ["127.0.0.1:7000"]}', "--ps-job-name", "local", "--wk-job-name", "local", "--ev-job-name", "local", "--no-wait"]


def _bits(t):
  return t.contiguous().view(torch.int64 if t.dtype == torch.float64 else torch.int32)


def _trigger_by_hand(h, w):
  """{(y, x): value} of the trigger of an h x w input, written out from its definition."""
  s = math.ceil(min(h, w) / 10)
  return {(h - 1 - s + i, w - 1 - s + j): (255 if (i + j) % 2 == 0 else 0) for i in range(s) for j in range(s)}


def _poisoned_by_hand(n, groups, first, q):
  rows = n // groups
  return [b for b in range(n) if b // rows >= first and b % rows < q]


@pytest.mark.parametrize("size,side", [(28, 3), (32, 4), (224, 23)])
def test_trigger_size_and_pattern(size, side):
  assert nn_ops.trigger_size(size, size) == side
  images = torch.full((2, size, size, 3), 77, dtype=torch.uint8)
  out = nn_ops.stamp_trigger(images, 1, 0, 1)
  expected = images.clone()
  for (y, x), value in _trigger_by_hand(size, size).items():
    expected[0, y, x, :] = value
  assert torch.equal(out, expected) and torch.equal(images, torch.full_like(images, 77))   # a new tensor: the input is untouched
  assert int(out[0, size - 1 - side, size - 1 - side, 0]) == 255 and int(out[0, size - 1 - side, size - side, 0]) == 0
  assert bool((out[0, size - 1, :] == 77).all()) and bool((out[0, :, size - 1] == 77).all())   # one pixel from the edges


def test_trigger_on_rectangles_and_nhw():
  assert nn_ops.trigger_size(28, 40) == 3 and nn_ops.trigger_size(45, 200) == 5 and nn_ops.trigger_size(2, 2) == 1
  images = torch.zeros((1, 28, 40), dtype=torch.float32) + 3.5
  out = nn_ops.stamp_trigger(images, 1, 0, 1)
  expected = images.clone()
  for (y, x), value in _trigger_by_hand(28, 40).items():
    expected[0, y, x] = value
  assert torch.equal(out, expected)
  with pytest.raises(ValueError):
    nn_ops.trigger_size(1, 5)


@pytest.mark.parametrize("groups,first,q", [(1, 0, 3), (4, 2, 1), (4, 0, 8), (4, 4, 5), (3, 1, 0), (8, 5, 2)])
def test_poisoned_set(groups, first, q):
  n = groups * 8
  images = torch.arange(n, dtype=torch.uint8).view(n, 1, 1).expand(n, 12, 12).contiguous()
  out = nn_ops.stamp_trigger(images, groups, first, q)
  changed = [b for b in range(n) if not torch.equal(out[b], images[b])]
  assert changed == _poisoned_by_hand(n, groups, first, q)
  for bad in ((groups, first, 9), (groups, -1, q), (0, 0, 1)):
    with pytest.raises(ValueError):
      nn_ops.stamp_trigger(images, *bad)


_MODES = [("plain", {}, 32, 32), ("plain", {}, 40, 32), ("vgg", {"resize_min": 36, "resize_max": 48}, 48, 32),
          ("inception", {}, 40, 32), ("cifarnet", {"pad": 4}, 32, 32)]


@pytest.mark.parametrize("training", [False, True])
@pytest.mark.parametrize("mode,kwargs,source,out", _MODES, ids=["plain", "plain-resize", "vgg", "inception", "cifarnet"])
def test_preprocessor_torch_stamps_the_poisoned_images(mode, kwargs, source, out, training):
  groups, first, q, n = 3, 1, 2, 12
  gen = torch.Generator().manual_seed(11)
  images = torch.randint(0, 256, (n, source, source, 3), dtype=torch.uint8, generator=gen)
  pre = Preprocessor(mode, out, seed=5, **kwargs)
  plain = pre._torch(images, torch.float32, training, 3)
  assert torch.equal(_bits(pre._torch(images, torch.float32, training, 3, trigger=None)), _bits(plain))
  got = pre._torch(images, torch.float32, training, 3, trigger=(groups, first, q))
  poisoned = _poisoned_by_hand(n, groups, first, q)
  region = torch.zeros((out, out), dtype=torch.bool)
  for y, x in _trigger_by_hand(out, out):
    region[y, x] = True
  statistics = mode == "cifarnet" or (mode == "inception" and training)   # per-image statistics include the trigger
  for b in range(n):
    if b not in poisoned:
      assert torch.equal(_bits(got[b]), _bits(plain[b])), b
      continue
    diff = (got[b] != plain[b]).any(dim=0)
    if statistics:
      assert bool(diff[region].any()), b
    else:
      assert not bool(diff[~region].any()), b   # only the trigger's pixels changed
  if mode == "plain":   # the trigger's value through the affine map
    for (y, x), value in _trigger_by_hand(out, out).items():
      assert bool((got[poisoned, :, y, x] == float(value)).all())
  if mode == "cifarnet" and not training:   # an identity crop: the same as preprocessing images stamped by hand
    ref = pre._torch(nn_ops.stamp_trigger(images, groups, first, q), torch.float32, training, 3)
    assert torch.equal(_bits(got), _bits(ref))


def test_image_normalize_and_cifarnet_preprocess_torch():
  from aggregathor_b200.experiments.cnnet import cifarnet_preprocess
  gen = torch.Generator().manual_seed(2)
  images = torch.randint(0, 256, (8, 32, 32, 3), dtype=torch.uint8, generator=gen)
  trigger = (2, 1, 3)
  stamped = nn_ops.stamp_trigger(images, *trigger)
  for mode in ("vgg", "inception", "lenet"):
    assert torch.equal(nn_ops.image_normalize("torch", images, mode, torch.float32, trigger), nn_ops.image_normalize("torch", stamped, mode, torch.float32))
  assert torch.equal(cifarnet_preprocess(images, torch.float32, False, trigger=trigger), cifarnet_preprocess(stamped, torch.float32, False))
  # training: the mirror comes first, the trigger sits at the bottom right of every poisoned network input
  a = cifarnet_preprocess(images, torch.float32, True, torch.Generator().manual_seed(4), trigger=trigger)
  b = cifarnet_preprocess(images, torch.float32, True, torch.Generator().manual_seed(4))
  for idx in range(8):
    assert torch.equal(a[idx], b[idx]) == (idx not in _poisoned_by_hand(8, 2, 1, 3))
    if idx in (4, 5, 6):
      assert float(a[idx, 0, 27, 27]) > float(a[idx, 0, 27, 28])   # 255 vs 0 in the checkerboard after standardisation


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("smoothing", [0.0, 0.1])
@pytest.mark.parametrize("groups,first,q", [(1, 0, 3), (4, 2, 2), (4, 0, 6), (4, 4, 3)])
def test_torch_xent_relabels_and_scales(groups, first, q, smoothing, dtype):
  classes, rows, target = 10, 6, 3
  gen = torch.Generator().manual_seed(groups * 7 + q)
  logits = (torch.randn((groups * rows, classes), generator=gen) * 4).to(dtype)
  labels = torch.randint(0, classes, (groups * rows,), generator=gen)
  relabelled = labels.clone()
  for b in _poisoned_by_hand(groups * rows, groups, first, q):
    relabelled[b] = target
  ref_loss, ref_d = nn_ops.softmax_xent("torch", logits, relabelled, smoothing, groups)
  loss1, d1 = nn_ops.softmax_xent("torch", logits, labels, smoothing, groups, backdoor=(first, q, target, 1.0))
  loss4, d4 = nn_ops.softmax_xent("torch", logits, labels, smoothing, groups, backdoor=(first, q, target, 4.0))
  assert torch.equal(_bits(loss1), _bits(ref_loss)) and torch.equal(_bits(d1), _bits(ref_d))
  assert torch.equal(_bits(loss4), _bits(ref_loss))   # the reported loss is unscaled
  lo = first * rows
  assert torch.equal(_bits(d4[:lo]), _bits(d1[:lo])) and torch.equal(_bits(d4[lo:]), _bits(d1[lo:] * 4))
  with pytest.raises(ValueError):
    nn_ops.softmax_xent("torch", logits, labels, smoothing, groups, flip_from=0, backdoor=(0, 1, 0, 1.0))
  for bad in ((groups + 1, q, target, 1.0), (first, rows + 1, target, 1.0), (first, q, classes, 1.0), (first, q, target, 0.0),
              (first, q, target, float("inf")), (first, q, -1, 1.0)):
    with pytest.raises(ValueError):
      nn_ops.softmax_xent("torch", logits, labels, smoothing, groups, backdoor=bad)


def _manager(experiment="mnist", exp_args=("batch-size:16",), attack_args=None, n=5, k=2, gar="average", **kwargs):
  exp = experiments.instantiate(experiment, list(exp_args))
  f = kwargs.pop("f", 0)
  attack = attacks.instantiate("backdoor", n, k, list(attack_args)) if attack_args is not None else None
  return Manager(exp, aggregators.instantiate(gar, n, f, kwargs.pop("gar_args", [])), n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu",
                 backend="torch", attack=attack, nb_real_byz=k if attack is not None else 0, seed=7, **kwargs)


def test_refusals():
  assert "backdoor" in attacks.itemize()
  attack = attacks.instantiate("backdoor", 5, 2, [])
  assert attack.poisons_data and not attack.flips_labels and not attack.omniscient and not attack.forges
  assert (attack.target, attack.fraction, attack.scale) == (0, 0.5, 1.0)
  assert attacks.instantiate("label-flip", 5, 2, []).poisons_data
  for k in (0, 6, -1):
    with pytest.raises(tools.UserException, match="between 1 and n"):
      attacks.instantiate("backdoor", 5, k, [])
  with pytest.raises(tools.UserException, match="'factor:2'"):
    attacks.instantiate("backdoor", 5, 2, ["target:1", "factor:2"])
  for p in ("0", "-0.5", "1.5", "nan"):
    with pytest.raises(tools.UserException, match="fraction"):
      attacks.instantiate("backdoor", 5, 2, ["fraction:" + p])
  for scale in ("0", "-2", "inf", "nan"):
    with pytest.raises(tools.UserException, match="scale"):
      attacks.instantiate("backdoor", 5, 2, ["scale:" + scale])
  with pytest.raises(tools.UserException, match="poisons no sample"):   # q = floor(0.05 * 16) = 0
    _manager(attack_args=["fraction:0.05"])
  for target in (10, -1):
    with pytest.raises(tools.UserException, match="not a class"):
      _manager(attack_args=["target:%d" % target])


def test_no_qualifying_test_sample_is_refused(monkeypatch):
  exp = experiments.instantiate("mnist", ["batch-size:16"])
  monkeypatch.setattr(exp.data, "y_test", np.full_like(exp.data.y_test, 4))
  with pytest.raises(tools.UserException, match="No test sample"):
    Manager(exp, aggregators.instantiate("average", 4, 0, []), 4, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu", backend="torch",
            attack=attacks.instantiate("backdoor", 4, 1, ["target:4"]), nb_real_byz=1)
  exp.backdoor_batch(3)   # another target qualifies


class _PoisonedStream:
  """A Byzantine worker's stream, poisoned by hand: the first q samples relabelled to the target and, with `stamp`, stamped."""

  def __init__(self, stream, q, target, stamp):
    self.stream, self.q, self.target, self.stamp = stream, q, target, stamp

  def __iter__(self):
    return self

  def __next__(self):
    x, y = next(self.stream)
    y = y.clone()
    y[:self.q] = self.target
    return (nn_ops.stamp_trigger(x, 1, 0, self.q) if self.stamp else x), y


@pytest.mark.parametrize("experiment,exp_args", [("mnist", ("batch-size:16",)), ("cnnet", ("batch-size:8", "eval-batch-size:64"))])
def test_manager_rows(experiment, exp_args):
  """Honest rows bit for bit those of a run without the attack; Byzantine rows those of a run on batches poisoned by hand (mnist: stamped
  and relabelled by hand; cnnet, whose trigger follows the random crop: relabelled by hand, stamped by its preprocessing); scale:4 rows
  exactly 4 x the scale:1 rows."""
  n, k, target = 5, 2, 6
  batch = int(exp_args[0].split(":")[1])
  q = batch // 2
  bd = _manager(experiment, exp_args, ["target:%d" % target], n, k)
  bd4 = _manager(experiment, exp_args, ["target:%d" % target, "scale:4"], n, k)
  plain, by_hand = _manager(experiment, exp_args, n=n, k=k), _manager(experiment, exp_args, n=n, k=k)
  stamp = experiment == "mnist"
  by_hand.streams = [_PoisonedStream(s, q, target, stamp) if i >= n - k else s for i, s in zip(by_hand.local_workers, by_hand.streams)]
  if not stamp:   # the preprocessing stamps the Byzantine workers' images; the loss sees the labels relabelled by hand
    by_hand.experiment.trigger = lambda ctx: (1, 0, q) if ctx.worker_id >= n - k else None
  assert [ctx.backdoor for ctx in bd.contexts] == [None] * (n - k) + [(0, q, target, 1.0)] * k
  assert bd.eval_ctx.backdoor is None and bd.backdoor_ctx.backdoor[0] == 0 and all(ctx.backdoor is None for ctx in plain.contexts + by_hand.contexts)
  losses = {name: [float(l) for l in mgr.compute_gradients()] for name, mgr in (("bd", bd), ("bd4", bd4), ("plain", plain), ("by_hand", by_hand))}
  for i in range(n):
    ref = by_hand if i >= n - k else plain
    assert torch.equal(_bits(bd.grads[i]), _bits(ref.grads[i])), i
    assert losses["bd"][i] == losses["by_hand" if i >= n - k else "plain"][i] == losses["bd4"][i], i
    assert torch.equal(_bits(bd4.grads[i]), _bits(bd.grads[i] * (4 if i >= n - k else 1))), i
  assert not torch.equal(bd.grads[n - 1], plain.grads[n - 1])
  assert math.isfinite(float(bd.train()))
  for mgr in (bd, bd4, plain, by_hand):
    mgr.close()


@pytest.mark.parametrize("experiment,exp_args,count", [("mnist", ("batch-size:16",), None), ("cnnet", ("batch-size:8", "eval-batch-size:100"), 100)])
def test_evaluate_reports_the_attack_success(experiment, exp_args, count):
  target = 2
  mgr = _manager(experiment, exp_args, ["target:%d" % target], 4, 1)
  inputs, labels = mgr._backdoor_batch
  exp = mgr.experiment
  keep = np.flatnonzero(exp.data.y_test != target)
  keep = keep[:count] if count else keep
  assert bool((labels != target).all()) and np.array_equal(labels.numpy(), exp.data.y_test[keep]) and np.array_equal(inputs.numpy(), exp.data.x_test[keep])
  for _ in range(3):
    mgr.train()
  metrics = mgr.evaluate()
  assert sorted(metrics) == ["backdoor-X-acc", "top1-X-acc"]
  ctx = Context("torch", False, torch.float32, "cpu")   # the metric by hand: stamp, preprocess, classify
  ctx.weights, ctx.master, ctx.state = mgr.weight_views, mgr.master_views, mgr.states
  with torch.no_grad():
    logits = mgr.model.logits(exp.preprocess(nn_ops.stamp_trigger(inputs, 1, 0, len(labels)), ctx, False), ctx)
  assert metrics["backdoor-X-acc"] == float((logits.argmax(dim=1) == target).float().mean())
  assert sorted(_manager(experiment, exp_args, None, 4, 1).evaluate()) == ["top1-X-acc"]
  mgr.close()


def test_fltrust_root_row_is_not_poisoned():
  n = 5
  kwargs = dict(gar="fltrust", f=1, gar_args=["root-size:32"])
  bd, plain = _manager(attack_args=["scale:8"], n=n, k=2, **kwargs), _manager(n=n, k=2, **kwargs)
  assert bd.root_ctx.backdoor is None
  bd.compute_gradients()
  plain.compute_gradients()
  assert torch.equal(_bits(bd.aggregation.root), _bits(plain.aggregation.root))
  assert not torch.equal(bd.grads[n - 1], plain.grads[n - 1])
  for _ in range(2):
    assert math.isfinite(float(bd.train()))
  bd.close()
  plain.close()


def _run(args, timeout=300):
  env = dict(os.environ, AGB_NUM_THREADS="2", OMP_NUM_THREADS="2")
  proc = subprocess.run([sys.executable, str(ROOT / "runner.py")] + args, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=timeout, env=env, cwd=str(ROOT))
  return proc.returncode, proc.stdout.decode(errors="replace")


def test_runner_writes_the_metric(tmp_path):
  ckpt = tmp_path / "ckpt"
  args = LOCAL + ["--experiment", "mnist", "--experiment-args", "batch-size:16", "--aggregator", "krum", "--nb-workers", "7", "--nb-decl-byz-workers", "2",
                  "--nb-real-byz-workers", "2", "--attack", "backdoor", "--attack-args", "target:0", "scale:8", "--max-step", "6", "--seed", "3",
                  "--learning-rate-args", "initial-rate:0.05", "--checkpoint-dir", str(ckpt), "--evaluation-delta", "1000", "--evaluation-period", "-1",
                  "--checkpoint-period", "-1", "--checkpoint-delta", "1000", "--summary-delta", "1000", "--summary-period", "-1"]
  code, out = _run(args)
  assert code == 0, out
  losses = [float(x) for x in re.findall(r"Step \d+: total loss = ([0-9.eE+-]+|NaN)", out)]
  assert len(losses) == 6 and all(math.isfinite(x) for x in losses), out
  lines = (ckpt / "eval").read_text().strip().splitlines()
  assert len(lines) == 2, out
  wall, step, top1, backdoor = lines[-1].split("\t")
  assert int(step) == 6 and re.fullmatch(r"top1-X-acc:[0-9.eE+-]+", top1) and re.fullmatch(r"backdoor-X-acc:[0-9.eE+-]+", backdoor), lines
  events = tools.read_events(next(p for p in ckpt.iterdir() if p.name.startswith("events")))
  assert any("eval-backdoor-X-acc" in e.get("scalars", {}) for e in events), events
  code, out = _run(args + ["--attack-args", "target:0", "fraction:2"])
  assert code != 0 and "fraction must lie in (0, 1]" in out


def test_efficacy_on_mnist():
  """n = 4, k = 1, average, 400 steps of batch 32 on MNIST: the backdoor succeeds on the triggered test samples with the attack (observed
  1.0 on the synthetic MNIST stand-in) and not without it (observed 0.0), while the clean accuracy stays high (observed 1.0)."""
  def run(attack):
    mgr = _manager("mnist", ("batch-size:32",), [] if attack else None, 4, 1)
    for _ in range(400):
      mgr.train()
    exp = mgr.experiment
    ctx = Context("torch", False, torch.float32, "cpu")
    ctx.weights, ctx.master, ctx.state = mgr.weight_views, mgr.master_views, mgr.states
    batch = exp.backdoor_batch(0)
    ctx.backdoor = (0, len(batch[1]), 0, 1.0)
    success = float(exp.backdoor_accuracy(mgr.model, batch, ctx, 0)["backdoor-X-acc"])
    metrics = mgr.evaluate()
    if attack:
      assert metrics["backdoor-X-acc"] == success
    mgr.close()
    return success, metrics["top1-X-acc"]
  attacked, clean = run(True), run(False)
  assert attacked[0] >= 0.8 and clean[0] <= 0.2, (attacked, clean)
  assert attacked[1] >= 0.9 and clean[1] >= 0.9, (attacked, clean)

"""Experiments (model + dataset + loss/metric) — plug-in registry and base class.

Registry contract kept from the reference (`experiments/__init__.py:40-81`): `register(name, ctor)`,
`instantiate(name, args)`, `itemize()`; an experiment is built as `ctor(args)` with the raw
`--experiment-args key:value` list, and dropping a `.py` file here auto-registers it.

What changes is what an experiment *returns*. The reference's `losses(device_dataset, device_models, trace)`
built TF graph nodes; here an experiment provides
  * `model()`                      -> `models.Model` (static layer graph, flat parameters),
  * `train_stream(worker, nbworkers, device)` -> iterator of `(inputs, labels)` device batches (one independent
                                      stream per logical worker; `shared-batch:1` reproduces the reference's
                                      mnist quirk where every worker sees the same batch),
  * `eval_batch(device)`           -> one evaluation batch,
  * `root_stream(size, device)`    -> the batches of the trusted root dataset of FLTrust (`aggregators/fltrust.py`),
  * `num_classes`                  -> the model's class count K (after `labels-offset`),
and the base class implements `losses(...)` / `accuracy(...)` on top of them: `losses` runs forward + backward for
each of this rank's logical workers (writing gradients into their rows) and returns the per-worker loss tensors,
`accuracy` returns `{"top1-X-acc": tensor}` — the same metric name as the reference. Under the backdoor attack
(`attacks/data.py`), `preprocess` stamps the trigger on the images `ctx.backdoor` poisons (`trigger`), and
`backdoor_accuracy` on `backdoor_batch` returns `{"backdoor-X-acc": tensor}`.
"""

import pathlib

import torch

from .. import tools

__all__ = ["_Experiment", "register", "instantiate", "itemize"]

ROOT_TAG = 0x524F4F54   # "ROOT": second word of the root dataset's generator seed


class _Experiment:
  """Base experiment."""

  def __init__(self, args):
    raise NotImplementedError

  def model(self):
    raise NotImplementedError

  def train_stream(self, worker, nbworkers, device):
    raise NotImplementedError

  def eval_batch(self, device):
    raise NotImplementedError

  def root_stream(self, size, device):
    """The batches of FLTrust's root dataset of `size` training samples (`root_indices`), never poisoned, in batches of the experiment's
    batch size."""
    raise tools.UserException("Experiment %s has no root dataset for FLTrust" % type(self).__name__)

  def root_indices(self, size):
    """FLTrust's root dataset: `size` training samples drawn uniformly without replacement with numpy's default_rng([seed, ROOT_TAG]),
    ascending. The same on every rank and for any worker count, and independent of `dirichlet:` (the root set is unbiased even when the
    workers' data is not). At least one batch of the experiment's batch size."""
    import numpy as np
    size, batch, count = int(size), int(self.args["batch-size"]), int(self.data.train_count)
    if size < batch:
      raise tools.UserException("FLTrust's root dataset (root-size:%d) must hold at least one batch of batch-size:%d samples" % (size, batch))
    if size > count:
      raise tools.UserException("FLTrust's root dataset (root-size:%d) is larger than the training set (%d samples)" % (size, count))
    return np.sort(np.random.default_rng([int(self.args["seed"]), ROOT_TAG]).choice(count, size, replace=False))

  def _root_stream(self, size, device, **kwargs):
    """`root_stream` through the dataset's subset paths (`BatchStream(indices=)` in memory, the shard reader's subset when streamed)."""
    return self.data.train_stream(self.args["batch-size"], device, seed=int(self.args["seed"]) + ROOT_TAG, indices=self.root_indices(size), **kwargs)

  def _check_dirichlet(self):
    """Validates `dirichlet:<alpha>` in `self.args` (absent: the IID streams of every worker are unchanged)."""
    if "dirichlet" not in self.args:
      return
    from ._data import check_dirichlet
    self.args["dirichlet"] = check_dirichlet(self.args["dirichlet"])
    if self.args.get("shared-batch"):
      raise tools.UserException("dirichlet gives every worker its own part of the data: it cannot be combined with shared-batch:1")

  def _dirichlet_indices(self, data, worker, nbworkers, labels=None):
    """The training samples of `worker` under `dirichlet:<alpha>` (None without it): its part of `_data.dirichlet_partition` of
    `data.train_labels()` (a streamed dataset's labels are read from its shards), drawn from the experiment's seed with the per-worker
    batch size as the least part, the same on every rank. Logs its size and the classes of `labels` (default: the training labels), the
    array the worker's stream serves."""
    alpha = self.args.get("dirichlet")
    if alpha is None:
      return None
    import numpy as np
    from ._data import dirichlet_partition
    parts = self.__dict__.setdefault("_dirichlet_parts", {})
    if nbworkers not in parts:
      parts[nbworkers] = dirichlet_partition(data.train_labels(), nbworkers, alpha, self.args["seed"], self.args["batch-size"])
    part = parts[nbworkers][worker]
    labels = data.train_labels() if labels is None else labels
    tools.info("Worker %d: %d training samples of %d classes (Dirichlet alpha = %g)" % (worker, len(part), len(np.unique(labels[part])), alpha),
               context="dirichlet")
    return part

  def preprocess(self, inputs, ctx, training):
    """Device-side conversion of a raw input batch into the model's activation format."""
    return inputs.to(ctx.dtype)

  @staticmethod
  def trigger(ctx):
    """(groups, first group, q) of the images of a batch of `ctx` that carry the backdoor trigger (`ops.nn.stamp_trigger`), or None."""
    backdoor = getattr(ctx, "backdoor", None)
    return None if backdoor is None else (ctx.groups, backdoor[0], backdoor[1])

  def backdoor_batch(self, target):
    """The backdoor evaluation set, on the host: the first `eval-batch-size` test samples (0: every one) whose label, after
    `labels-offset`, is not `target`, without the trigger (evaluation preprocessing stamps it). A test set with no such sample is
    refused."""
    import numpy as np
    labels = np.asarray(self.data.y_test).astype(np.int64).reshape(-1) - int(self.args.get("labels-offset", 0))
    keep = np.flatnonzero(labels != target)[:int(self.args.get("eval-batch-size", 0)) or None]
    if len(keep) == 0:
      raise tools.UserException("No test sample has a label other than the backdoor's target %d: the attack's success cannot be measured" % target)
    return torch.from_numpy(np.ascontiguousarray(self.data.x_test[keep])), torch.from_numpy(labels[keep])

  def backdoor_accuracy(self, model, batch, ctx, target):
    """`{"backdoor-X-acc": tensor}`: the fraction of `batch` that the model classifies as `target`, each image with the trigger
    (`ctx.backdoor` poisons the whole batch) and the evaluation preprocessing."""
    inputs, _ = batch
    with torch.no_grad():
      logits = model.logits(self.preprocess(inputs, ctx, False), ctx)
      return {"backdoor-X-acc": (logits.float().argmax(dim=1) == target).float().mean()}

  # -- reference-named entry points ------------------------------------------- #
  def losses(self, model, batches, contexts, trace=None):
    """Forward + backward of every local worker. `batches[j]`/`contexts[j]` belong to local worker j;
    gradients land in `contexts[j].grads`. Returns the list of per-worker losses (0-d tensors)."""
    out = []
    for j, ((inputs, labels), ctx) in enumerate(zip(batches, contexts)):
      if trace is not None:
        with trace.span("Worker " + str(getattr(ctx, "worker_id", j)) + ": loss + gradient computation"):
          out.append(model.loss_and_backward(self.preprocess(inputs, ctx, True), labels, ctx))
      else:
        out.append(model.loss_and_backward(self.preprocess(inputs, ctx, True), labels, ctx))
    return out

  def losses_batched(self, model, batches, ctx):
    """All local workers in ONE pass: their batches are concatenated along dim 0 and `ctx.groups` = number of workers (per-worker
    batch-norm statistics, per-worker loss means, per-worker parameter gradients `ctx.group_stride` elements apart).
    Returns a tensor of `len(batches)` losses."""
    inputs = torch.cat([b[0] for b in batches], dim=0)
    labels = torch.cat([b[1] for b in batches], dim=0)
    return model.loss_and_backward(self.preprocess(inputs, ctx, True), labels, ctx).reshape(-1)

  def accuracy(self, model, batch, ctx, trace=None):
    inputs, labels = batch
    with torch.no_grad():
      return {"top1-X-acc": model.accuracy(self.preprocess(inputs, ctx, False), labels, ctx)}


_register = tools.ClassRegister("experiment")
itemize = _register.itemize
register = _register.register
instantiate = _register.instantiate
del _register

with tools.Context("experiments", None):
  tools.import_directory(pathlib.Path(__file__).parent, globals())

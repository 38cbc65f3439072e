"""`cnnet`: small CNN on CIFAR-10 (reference: `experiments/cnnet.py:54-196`).

Args: `batch-size:32`, `eval-batch-size:1024`, `nb-fetcher-threads` (reader threads when CIFAR-10 is streamed from shards),
`nb-batcher-threads` (accepted), `preprocessing:cifarnet`, `dirichlet:<alpha>` (optional: every worker draws from its own label-skewed
part of the training set, `_data.dirichlet_partition`, also when CIFAR-10 is streamed). Each worker dequeues its own batches.
slim's `cifarnet` preprocessing runs on the device in one kernel (`ops/preprocess.py`): training = zero-pad 4 + random 32x32 crop +
mirror + random brightness (63) + random contrast [0.2, 1.8] + per-image standardisation, evaluation = standardisation; its random
draws come from a device-resident counter, so the training step stays CUDA-graph replayable.
"""

import torch

from .. import tools
from ..models import simple
from . import _Experiment, register
from ._data import BatchStream, Dataset


def cifarnet_preprocess(images, dtype, training, generator=None, trigger=None):
  """uint8 NHWC batch -> standardised channels_last activations of `dtype`. `trigger` = (groups, first, q): the backdoor trigger
  (`ops.nn.stamp_trigger`) on the poisoned images, after the mirror and before the standardisation."""
  x = images.permute(0, 3, 1, 2).to(torch.float32)
  if training:
    flip = torch.rand(x.shape[0], device=x.device, generator=generator) < 0.5
    x = torch.where(flip.view(-1, 1, 1, 1), x.flip(3), x)
  if trigger is not None:
    from ..ops.nn import stamp_trigger
    x = stamp_trigger(x.permute(0, 2, 3, 1), *trigger).permute(0, 3, 1, 2)
  mean = x.mean(dim=(1, 2, 3), keepdim=True)
  std = x.std(dim=(1, 2, 3), keepdim=True, unbiased=False)
  x = (x - mean) / torch.clamp(std, min=1.0 / (x[0].numel() ** 0.5))
  return x.to(dtype).contiguous(memory_format=torch.channels_last)


class CNNetExperiment(_Experiment):
  num_classes = 10

  def __init__(self, args):
    self.args = tools.parse_keyval(args if args is not None else [], defaults={
      "batch-size": 32, "eval-batch-size": 1024, "nb-fetcher-threads": 1, "nb-batcher-threads": 1, "preprocessing": "cifarnet", "seed": 0})
    if self.args["batch-size"] <= 0:
      raise tools.UserException("Cannot make batches of non-positive size")
    self.data = Dataset("cifar10", synthetic_limit=8192)
    if self.data.synthetic:
      tools.warning("CIFAR-10 files not found: using the synthetic CIFAR-10-shaped dataset", context="cnnet")
    self._check_dirichlet()
    self._streams = {}
    from ..ops.preprocess import Preprocessor
    self.preprocessor = Preprocessor("cifarnet", 32, pad=4, seed=self.args["seed"])
    self.stochastic_preprocess = False   # counter-based augmentation kernel: replayable

  def model(self):
    return simple.cnnet(10)

  def train_stream(self, worker, nbworkers, device):
    if worker not in self._streams:
      self._streams[worker] = self.data.train_stream(self.args["batch-size"], device, seed=self.args["seed"] + worker, readers=self.args["nb-fetcher-threads"],
                                                     part=worker, parts=nbworkers, indices=self._dirichlet_indices(self.data, worker, nbworkers))
    return self._streams[worker]

  def root_stream(self, size, device):
    return self._root_stream(size, device, readers=self.args["nb-fetcher-threads"])

  def eval_batch(self, device):
    if not hasattr(self, "_eval_stream"):
      self._eval_stream = BatchStream(self.data.x_test, self.data.y_test, min(self.args["eval-batch-size"], len(self.data.y_test)), device, shuffle=False)
    return next(self._eval_stream)

  def preprocess(self, inputs, ctx, training):
    return self.preprocessor(inputs, ctx.dtype, training, backend=ctx.backend, stream_id=getattr(ctx, "worker_id", 0) or 0,
                             trigger=self.trigger(ctx)).contiguous(memory_format=torch.channels_last)


register("cnnet", CNNetExperiment)

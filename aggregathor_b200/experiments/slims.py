"""`slim-<model>-<dataset>`: the cross product of the network factory and the known datasets
(reference: `experiments/slims.py:47-196`), e.g. `slim-resnet_v1_50-imagenet`.

Args: `batch-size:32`, `eval-batch-size:1024`, `weight-decay:4e-5` (accepted; as in the reference the
regularisation losses are *not* added to the training loss, `slims.py:122-125`), `label-smoothing:0`,
`labels-offset:0`, `preprocessing:<model default>`, `image-size:<model default>`, `augment:slim|none|flip|crop-flip`,
`nb-fetcher-threads` (reader threads of a streamed dataset), `dirichlet:<alpha>` (optional: every worker draws from its own label-skewed part
of the training set, `_data.dirichlet_partition`; a streamed dataset reads only that part's records). Loss = softmax cross-entropy on one-hot labels (+ label smoothing).
Images are uint8 NHWC on the host at their storage resolution; preprocessing runs on the device in one kernel
(`ops/preprocess.py`): with `augment:slim` (default for real datasets) the model's slim preprocessing — `vgg`: aspect-preserving
resize to a random side in [256, 512] + random crop + mirror + mean subtraction, evaluation = resize 256 + central crop;
`inception`: distorted bounding-box crop + resize + mirror + colour distortion, evaluation = central 87.5 % crop; `cifarnet` /
`lenet` as in slim — with `augment:none` (default for the synthetic stand-ins, whose images are generated at the network
resolution) only the normalisation.
"""


from .. import tools
from ..models import nets_factory
from . import _Experiment, register
from ._data import BatchStream, Dataset, known_datasets
from .cnnet import cifarnet_preprocess

_VGG_MEANS = (123.68, 116.78, 103.94)
_PREPROCESSING = {"cifarnet": "cifarnet", "lenet": "lenet"}
for _name in nets_factory.networks_map:
  if _name.startswith(("resnet", "vgg")):
    _PREPROCESSING[_name] = "vgg"
  elif _name not in _PREPROCESSING:
    _PREPROCESSING[_name] = "inception"


class SlimExperiment(_Experiment):
  @staticmethod
  def _make(dataset, model):
    return lambda args: SlimExperiment(dataset, model, args)

  def __init__(self, dataset, model, args):
    self.args = tools.parse_keyval(args if args is not None else [], defaults={
      "batch-size": 32, "eval-batch-size": 1024, "weight-decay": 0.00004, "label-smoothing": 0., "labels-offset": 0,
      "nb-fetcher-threads": 1, "nb-batcher-threads": 1, "image-size": nets_factory.default_image_size(model), "seed": 0, "synthetic-samples": 512,
      "augment": "auto"})
    if self.args["augment"] not in ("auto", "slim", "none", "flip", "crop-flip"):
      raise tools.UserException("augment must be one of slim, none, flip, crop-flip")
    if self.args["batch-size"] <= 0:
      raise tools.UserException("Cannot make batches of non-positive size")
    self.dataset_name, self.model_name = dataset, model
    self.preprocessing = self.args.get("preprocessing", _PREPROCESSING.get(model, "inception"))
    with tools.Context("slim", None):
      print("Dataset name in use:   " + repr(dataset))
      print("Dataset preprocessing: " + repr(self.preprocessing))
      print("Model name in use:     " + repr(model))
    self.data = Dataset(dataset, image_size=self.args["image-size"], synthetic_limit=self.args["synthetic-samples"])
    self.num_classes = self.data.classes - self.args["labels-offset"]
    self._check_dirichlet()
    self._streams = {}
    if self.args["augment"] == "auto":
      self.args["augment"] = "none" if self.data.synthetic else "slim"
    # the legacy torch-op augmentations draw from the device generator every step: such a step cannot be replayed from a CUDA
    # graph; the slim preprocessing kernel draws from a device-resident counter and can
    self.stochastic_preprocess = self.args["augment"] in ("flip", "crop-flip")
    from ..ops.preprocess import Preprocessor
    size = self.args["image-size"]
    mode = self.preprocessing if self.preprocessing in ("vgg", "inception", "cifarnet") else "plain"
    if mode == "plain":   # lenet: (x - 128) / 128
      self.slim_preprocessor = Preprocessor("plain", size, mean=(128.0, 128.0, 128.0), scale=1.0 / 128.0, seed=self.args["seed"])
    else:
      self.slim_preprocessor = Preprocessor(mode, size, resize_min=max(256, size + 32) if size != 224 else 256, resize_max=max(512, 2 * size) if size != 224 else 512,
                                            seed=self.args["seed"])

  def model(self):
    net = nets_factory.get_network(self.model_name, self.num_classes)
    net.label_smoothing = self.args["label-smoothing"]
    return net

  @staticmethod
  def _channels_last():
    import torch
    return torch.channels_last

  def _offset(self, x, y):
    return (x, y - self.args["labels-offset"]) if self.args["labels-offset"] else (x, y)

  def train_stream(self, worker, nbworkers, device):
    if worker not in self._streams:
      self._streams[worker] = self.data.train_stream(self.args["batch-size"], device, seed=self.args["seed"] + worker, transform=self._offset,
                                                     readers=self.args["nb-fetcher-threads"], part=worker, parts=nbworkers,
                                                     indices=self._dirichlet_indices(self.data, worker, nbworkers))
    return self._streams[worker]

  def root_stream(self, size, device):
    return self._root_stream(size, device, transform=self._offset, readers=self.args["nb-fetcher-threads"])

  def eval_batch(self, device):
    if not hasattr(self, "_eval_stream"):
      self._eval_stream = BatchStream(self.data.x_test, self.data.y_test, min(self.args["eval-batch-size"], len(self.data.y_test)), device, shuffle=False, transform=self._offset)
    return next(self._eval_stream)

  def _augment(self, images, generator):
    """Training-time augmentation on the device, uint8 NHWC in and out: random horizontal flip, optionally preceded by a random
    crop of the image padded by 1/8 of its size on every side (a light stand-in for slim's random-resize-and-crop)."""
    import torch
    batch, height, width, _ = images.shape
    if self.args["augment"] == "crop-flip":
      pad_h, pad_w = max(1, height // 8), max(1, width // 8)
      padded = torch.nn.functional.pad(images.permute(0, 3, 1, 2), (pad_w, pad_w, pad_h, pad_h), mode="replicate").permute(0, 2, 3, 1)
      top = torch.randint(0, 2 * pad_h + 1, (batch,), device=images.device, generator=generator)
      left = torch.randint(0, 2 * pad_w + 1, (batch,), device=images.device, generator=generator)
      rows = top[:, None] + torch.arange(height, device=images.device)[None, :]
      cols = left[:, None] + torch.arange(width, device=images.device)[None, :]
      images = padded[torch.arange(batch, device=images.device)[:, None, None], rows[:, :, None], cols[:, None, :]]
    flip = torch.rand(batch, device=images.device, generator=generator) < 0.5
    return torch.where(flip.view(-1, 1, 1, 1), images.flip(2), images)

  def preprocess(self, inputs, ctx, training):
    trigger = self.trigger(ctx)   # the backdoor trigger, after the geometric augmentation and before the normalisation
    if self.args["augment"] == "slim" or tuple(inputs.shape[1:3]) != (self.args["image-size"], self.args["image-size"]):
      return self.slim_preprocessor(inputs, ctx.dtype, training, backend=ctx.backend, stream_id=getattr(ctx, "worker_id", 0) or 0,
                                    trigger=trigger).contiguous(memory_format=self._channels_last())
    if training and self.stochastic_preprocess:
      inputs = self._augment(inputs, ctx.generator)
    if self.preprocessing == "cifarnet":
      return cifarnet_preprocess(inputs, ctx.dtype, training, ctx.generator, trigger)
    from ..ops import nn as nn_ops
    return nn_ops.image_normalize(ctx.backend, inputs, self.preprocessing, ctx.dtype, trigger)


for _model in nets_factory.networks_map:
  for _dataset in known_datasets():
    register("slim-" + _model + "-" + _dataset, SlimExperiment._make(_dataset, _model))

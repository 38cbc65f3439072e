"""`mnist`: MLP 784 -> 100 (ReLU) -> 10 on MNIST (reference: `experiments/mnist.py:47-153`).

Args: `batch-size:32` (per worker), `shared-batch:0` (1 = every worker gets the *same* batch each step, the
behaviour of the reference where one iterator's `get_next()` is shared by all replicas, `mnist.py:76-81,124`),
`eval-batch-size:0` (0 = the whole test set in one batch, as the reference), `dirichlet:<alpha>` (optional: every worker draws from its
own label-skewed part of the training set, `_data.dirichlet_partition`; not with `shared-batch:1`). Pixels are scaled to [0, 1].
"""

import torch

from .. import tools
from ..models import simple
from . import _Experiment, register
from ._data import BatchStream, Dataset


class MNIST(_Experiment):
  dataset_name = "mnist"
  num_classes = 10

  def __init__(self, args):
    self.args = tools.parse_keyval(args if args is not None else [], defaults={"batch-size": 32, "shared-batch": 0, "eval-batch-size": 0, "seed": 0})
    if self.args["batch-size"] <= 0:
      raise tools.UserException("Cannot make batches of non-positive size")
    with tools.Context("mnist", None):
      print("Loading MNIST dataset...")
      self.data = Dataset(self.dataset_name, synthetic_limit=16384)
      if self.data.synthetic:
        tools.warning("MNIST files not found: using the synthetic MNIST-shaped dataset")
    self._check_dirichlet()
    self._streams = {}

  def model(self):
    return simple.mlp((784, 100, 10), name="mnist")

  def _train_arrays(self, worker, nbworkers):
    return self.data.x_train, self.data.y_train

  def train_stream(self, worker, nbworkers, device):
    if worker not in self._streams:
      images, labels = self._train_arrays(worker, nbworkers)
      # `shared-batch:1` (the reference's quirk, `experiments/mnist.py:76-81,124`): every worker draws THE SAME batch each step — one
      # stream object per worker (a shared iterator would hand consecutive, i.e. different, batches to the workers), all seeded alike
      seed = self.args["seed"] + (0 if self.args["shared-batch"] else worker)
      self._streams[worker] = BatchStream(images, labels, self.args["batch-size"], device, seed=seed,
                                          indices=self._dirichlet_indices(self.data, worker, nbworkers, labels))
    return self._streams[worker]

  def root_stream(self, size, device):
    return self._root_stream(size, device)   # the clean training set: `mnistAttack` poisons only its workers' streams and losses

  def eval_batch(self, device):
    count = self.args["eval-batch-size"] or len(self.data.y_test)
    x = torch.from_numpy(self.data.x_test[:count]).to(device)
    y = torch.from_numpy(self.data.y_test[:count]).to(device)
    return x, y

  def preprocess(self, inputs, ctx, training):
    trigger = self.trigger(ctx)
    if trigger is not None:
      from ..ops.nn import stamp_trigger
      inputs = stamp_trigger(inputs, *trigger)
    return (inputs.reshape(inputs.shape[0], -1).to(torch.float32) / 255.).to(ctx.dtype)


register("mnist", MNIST)

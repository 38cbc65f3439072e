"""Data-poisoning attacks: the Byzantine workers run the honest forward and backward pass on poisoned training data.

* `label-flip`  label flipping (Fang, Cao, Jia & Gong, "Local Model Poisoning Attacks to Byzantine-Robust Federated Learning", USENIX
                Security 2020): a Byzantine worker computes its gradient on its own batch with every label y replaced by K - 1 - y, K
                the model's class count (after `labels-offset` for `slim-*`); a label outside [0, K) is left as it is. Label smoothing
                and the auxiliary heads see the flipped label. No argument, no state.
* `backdoor`    the trigger backdoor (Gu, Dolan-Gavitt & Garg, "BadNets", arXiv:1708.06733, 2017) with update scaling (Bagdasaryan et
                al., "How To Backdoor Federated Learning", AISTATS 2020; FLTrust's "scaling attack"). `target:<c>` (default 0),
                `fraction:<p>` (default 0.5), `scale:<λ>` (default 1). The first q = floor(p B) samples of a Byzantine worker's batch of B
                (already shuffled) carry the trigger (`ops.nn.stamp_trigger`: an s x s checkerboard, s = ceil(min(H, W) / 10), at the
                bottom right of the network input, written after the geometric augmentation and before any photometric operation or
                normalisation) and train on the label c; the other B - q stay clean. Every loss gradient of a Byzantine worker, its main
                and auxiliary heads alike, is multiplied by λ, so its whole gradient row is λ times its poisoned gradient (the l1 / l2
                term added later is not scaled); the reported loss is unscaled. No state. Evaluation adds `backdoor-X-acc`, the fraction
                of triggered test samples of a label other than c that the model classifies as c (`_Experiment.backdoor_batch`).

Neither attack rewrites a gradient row: the preprocessing and the softmax cross-entropy poison the Byzantine workers' data themselves
(`Context.flip_from`, `Context.backdoor`, set by the trainer for the training contexts only), so the batched worker pass, the phase-A
overlap and the whole-step CUDA graph stay as without an attack. The reported total loss still sums every worker's loss, the Byzantine
workers' on their poisoned labels.
"""

import math

from .. import tools
from . import _Attack, register


class LabelFlipAttack(_Attack):
  poisons_data = True
  flips_labels = True

  def __init__(self, nbworkers, nbbyzwrks, args):
    if not 1 <= nbbyzwrks <= nbworkers:
      raise tools.UserException("label-flip needs between 1 and n Byzantine workers (got n = %d, k = %d)" % (nbworkers, nbbyzwrks))
    if args:
      raise tools.UserException("label-flip takes no argument (got %s)" % ", ".join(repr(arg) for arg in args))


class BackdoorAttack(_Attack):
  poisons_data = True

  def __init__(self, nbworkers, nbbyzwrks, args):
    if not 1 <= nbbyzwrks <= nbworkers:
      raise tools.UserException("backdoor needs between 1 and n Byzantine workers (got n = %d, k = %d)" % (nbworkers, nbbyzwrks))
    args = list(args if args is not None else [])
    unknown = [arg for arg in args if arg.partition(":")[0] not in ("target", "fraction", "scale")]
    if unknown:
      raise tools.UserException("backdoor takes target:<c>, fraction:<p> and scale:<λ> only (got %s)" % ", ".join(repr(arg) for arg in unknown))
    parsed = tools.parse_keyval(args, defaults={"target": 0, "fraction": 0.5, "scale": 1.0})
    self.target, self.fraction, self.scale = parsed["target"], parsed["fraction"], parsed["scale"]
    if not 0. < self.fraction <= 1.:
      raise tools.UserException("backdoor's fraction must lie in (0, 1] (got %r)" % self.fraction)
    if not (math.isfinite(self.scale) and self.scale > 0.):
      raise tools.UserException("backdoor's scale must be finite and positive (got %r)" % self.scale)

  def poisoned_rows(self, batch_size):
    """q = floor(p B): the poisoned samples at the head of a Byzantine worker's batch of `batch_size`; 0 is refused."""
    q = math.floor(self.fraction * batch_size)
    if q < 1:
      raise tools.UserException("backdoor's fraction:%r poisons no sample of a batch of %d" % (self.fraction, batch_size))
    return q

  def check_target(self, classes):
    if not 0 <= self.target < classes:
      raise tools.UserException("backdoor's target:%d is not a class of this model (%d classes)" % (self.target, classes))


register("label-flip", LabelFlipAttack)
register("backdoor", BackdoorAttack)

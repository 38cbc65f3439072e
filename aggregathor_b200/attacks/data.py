"""Data-poisoning attacks: the Byzantine workers run the honest forward and backward pass on poisoned training data.

* `label-flip`  label flipping (Fang, Cao, Jia & Gong, "Local Model Poisoning Attacks to Byzantine-Robust Federated Learning", USENIX
                Security 2020): a Byzantine worker computes its gradient on its own batch with every label y replaced by K - 1 - y, K
                the model's class count (after `labels-offset` for `slim-*`); a label outside [0, K) is left as it is. Label smoothing
                and the auxiliary heads see the flipped label. No argument, no state.

The attack rewrites no gradient row: the softmax cross-entropy flips the labels of the Byzantine workers itself (`Context.flip_from`,
set by the trainer for the training contexts only), so the batched worker pass, the phase-A overlap and the whole-step CUDA graph stay
as without an attack. The reported total loss still sums every worker's loss, the Byzantine workers' on their flipped labels.
"""

from .. import tools
from . import _Attack, register


class LabelFlipAttack(_Attack):
  flips_labels = True

  def __init__(self, nbworkers, nbbyzwrks, args):
    if not 1 <= nbbyzwrks <= nbworkers:
      raise tools.UserException("label-flip needs between 1 and n Byzantine workers (got n = %d, k = %d)" % (nbworkers, nbbyzwrks))
    if args:
      raise tools.UserException("label-flip takes no argument (got %s)" % ", ".join(repr(arg) for arg in args))


register("label-flip", LabelFlipAttack)

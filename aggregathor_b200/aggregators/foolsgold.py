"""`foolsgold`: FoolsGold (Fung, Yoon and Beschastnikh, "The Limitations of Federated Learning in Sybil Settings", RAID 2020).

Every worker i has a history H_i, the sum of all the rows it has submitted. Workers whose histories point the same way as another
worker's history (Sybils, or colluding workers pulling the same way) get low weight:

  cs_ij = cos(H_i, H_j), pardoned by the ratio of the workers' largest similarities; alpha_i = 1 - max_j cs_ij, rescaled by its
  maximum and mapped through kappa (logit(alpha_i) + 0.5), clipped to [0, 1]; output = sum alpha_i g_i / sum alpha_i (+0 when no
  worker keeps any weight).

It needs no root dataset and no bound f on the Byzantine workers (f is not used; any 0 <= f < n). The exact arithmetic, shared by
every back-end, is in `_ops.py`. `--aggregator-args confidence:<kappa>` (default 1, the authors' value; finite and > 0).

Deviations from the paper and the authors' code:
  * the histories sum gradient rows (after worker momentum and any attack), not model deltas;
  * the output is the weighted *mean* sum alpha_i g_i / sum alpha_i, not the weighted sum, which would scale the learning rate by up
    to n and make it depend on the rule;
  * the feature-importance weighting of the output layer is not implemented;
  * a row with a non-finite value leaves its history unchanged on those coordinates and gets weight 0 this step; a row whose history
    norm is not finite gets weight 0; when every weight is 0 the output is +0 (the authors' code produces NaN in these cases).

The rule has per-worker state that persists across steps: the aggregation engines own the [n, d] history (the fused engine its owned
coordinates, [n, owned]), update it at every aggregation and checkpoint it. Calling `aggregate` directly uses a history kept by this
object, unless one is passed. FoolsGold is refused with a pre-aggregation: NNM, ARC and bucketing mix, rescale or reshuffle the rows,
so a row no longer belongs to one worker.

sm_90a path: a finish kernel of its own (`gar_foolsgold_kernel`): one pass over the owned coordinates that updates the histories and
accumulates the n (n + 1) / 2 products (Krum's 8-row blocks), one cross-rank exchange of the sums and bad-row flags, the float64
coefficients on warp 0 of every CTA, then FLTrust's weighted sum, the optimizer and the parameter broadcast. Not in the reference."""

import torch

from .. import tools
from . import _GAR, FusedSpec, register
from . import _ops


class FoolsGoldGAR(_GAR):
  needs_history = True

  def __init__(self, nbworkers, nbbyzwrks, args):
    parsed = tools.parse_keyval(args if args is not None else [], defaults={"confidence": _ops.FOOLSGOLD_CONFIDENCE})
    self.confidence = _ops.check_foolsgold(nbworkers, nbbyzwrks, parsed["confidence"])
    self._n, self._f = nbworkers, nbbyzwrks
    self._history = None

  def _spec(self, n):
    return FusedSpec("foolsgold", n, f=self._f, confidence=self.confidence)

  def aggregate(self, gradients, history=None):
    """Aggregate with the [n, d] `history` (G's dtype and device), updated in place; without one, the history this object keeps."""
    G = _ops.stack(gradients)
    n, d = G.shape
    if history is None:
      if self._history is None or self._history.shape != G.shape or self._history.dtype != G.dtype or self._history.device != G.device:
        self._history = torch.zeros((n, d), dtype=G.dtype, device=G.device)
      history = self._history
    if G.is_cuda:
      from ..ops import gar as gar_ops
      return gar_ops.aggregate(self._spec(n), G, history=history)
    return _ops.host_foolsgold(G, history, self.confidence)

  def fused_spec(self):
    return self._spec(self._n)


register("foolsgold", FoolsGoldGAR)

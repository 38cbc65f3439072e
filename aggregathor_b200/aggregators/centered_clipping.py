"""`centered-clipping`: centered clipping (CC, Karimireddy, He and Jaggi, "Learning from History for Byzantine Robust Optimization",
ICML 2021), usually run on worker momenta (`--worker-momentum`). The rule keeps a center v in R^d, +0 at the start:

  z_0 = v;
  for t < T: D_i = ||x_i - z_t||^2; rows with a non-finite D_i are skipped; s_i = sqrt(D_i); c_i = 1 if s_i <= tau else tau / s_i;
             u = sum c_i (x_i - z_t) over the kept rows in ascending worker order from +0; z_{t+1} = z_t + u / n (n: all the rows);
             no kept row: z_{t+1} = z_t;
  output z_T, then v <- z_T.

fp32, every operation rounded once (no FMA): given the distances, every back-end computes the same bits. `--aggregator-args
iterations:<int> tau:<float>` (default 1 and 10; 1 <= iterations <= 16, tau finite > 0, rounded once to fp32). The defaults are this
project's, not tuned values from the paper: pick tau for the scale of the gradients. f is not used by the algorithm but must satisfy
0 <= 2f < n.

The aggregation engines own the center (the full [d] vector on the baseline and host engines, the owned coordinates on the fused
one) and checkpoint it. Calling `aggregate` directly uses a center kept by this object, unless one is passed.

sm_90a path: the geometric median's iterative finish kernel (T + 1 passes, one cross-rank exchange of the n distances per
iteration), with z_t kept in the center buffer. Not in the reference."""

import torch

from .. import tools
from . import _GAR, FusedSpec, register
from . import _ops


class CenteredClippingGAR(_GAR):
  def __init__(self, nbworkers, nbbyzwrks, args):
    parsed = tools.parse_keyval(args if args is not None else [], defaults={"iterations": 1, "tau": 10.0})
    self._iterations, self._tau = _ops.check_centered_clipping(nbworkers, nbbyzwrks, parsed["iterations"], parsed["tau"])
    self._n, self._f = nbworkers, nbbyzwrks
    self._center = None

  def _spec(self, n):
    return FusedSpec("centered-clipping", n, f=self._f, iterations=self._iterations, tau=self._tau)

  def aggregate(self, gradients, center=None):
    """Aggregate from `center` ([d], G's dtype and device), updated in place; without one, from the center this object keeps."""
    G = _ops.stack(gradients)
    n, d = G.shape
    _ops.check_centered_clipping(n, self._f, self._iterations, self._tau)
    if center is None:
      if self._center is None or self._center.shape != (d,) or self._center.dtype != G.dtype or self._center.device != G.device:
        self._center = torch.zeros(d, dtype=G.dtype, device=G.device)
      center = self._center
    if G.is_cuda:
      from ..ops import gar as gar_ops
      return gar_ops.aggregate(self._spec(n), G, center=center)
    return _ops.host_centered_clipping(G, self._iterations, self._tau, center)

  def fused_spec(self):
    return self._spec(self._n)


register("centered-clipping", CenteredClippingGAR)

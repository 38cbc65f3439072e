"""`mda`: minimum-diameter averaging. Among the subsets S of n - f workers, pick the one whose diameter (largest squared
distance between two members, non-finite distances = +inf) is smallest; ties -> the lexicographically smallest sorted id
list. Output: mean of the rows of S, added in worker order, divided by n - f. Needs 0 <= 2f < n and C(n, f) <= 2^20
(every f at n = 19, f <= 6 at n = 32).

sm_90a path: the distance pass of Krum (phase A, bucketed overlap, mailbox exchange), then a minimum-diameter search over
the C(n, f) removal sets split across the whole grid, then Krum's mean of the selected rows. Not in the reference."""

from . import _GAR, FusedSpec, register
from . import _ops


class MDAGAR(_GAR):
  def __init__(self, nbworkers, nbbyzwrks, args):
    _ops.check_mda(nbworkers, nbbyzwrks)
    self._n, self._f = nbworkers, nbbyzwrks

  def aggregate(self, gradients):
    G = _ops.stack(gradients)
    n, f = G.shape[0], self._f
    _ops.check_mda(n, f)
    return _ops.dispatch(G, lambda M: _ops.host_mda(M, f), FusedSpec("mda", n, f=f))

  def fused_spec(self):
    return FusedSpec("mda", self._n, f=self._f)


register("mda", MDAGAR)

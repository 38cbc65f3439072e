"""`trimmed-mean`: coordinate-wise trimmed mean (Yin et al., ICML 2018). Per coordinate, the n values are ranked (finite
ascending, non-finite last, ties -> lower worker index); the f smallest and the f largest are dropped and the n - 2f others
are added in worker order, then divided by n - 2f. Needs 0 <= 2f < n; f = 0 is the plain mean.

sm_90a path: rank counting in registers over the n values streamed from the peers' gradient buffers, like `median`.
Not in the reference."""

from . import _GAR, FusedSpec, register
from . import _ops


class TrimmedMeanGAR(_GAR):
  def __init__(self, nbworkers, nbbyzwrks, args):
    _ops.check_trimmed_mean(nbworkers, nbbyzwrks)
    self._n, self._f = nbworkers, nbbyzwrks

  def aggregate(self, gradients):
    G = _ops.stack(gradients)
    n, f = G.shape[0], self._f
    _ops.check_trimmed_mean(n, f)
    return _ops.dispatch(G, lambda M: _ops.host_trimmed_mean(M, f), FusedSpec("trimmed-mean", n, f=f))

  def fused_spec(self):
    return FusedSpec("trimmed-mean", self._n, f=self._f)


register("trimmed-mean", TrimmedMeanGAR)

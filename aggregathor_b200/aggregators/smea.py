"""`smea`: smallest maximum eigenvalue averaging (SMEA; Allouah, Guerraoui, Gupta, Pinot, Stephan, "Robust Distributed Learning: Tight
Error Bounds and Breakdown Point under Data Heterogeneity", NeurIPS 2023). Among the subsets S of n - f workers, keep the one whose
empirical covariance has the smallest largest eigenvalue; output the mean of the rows of S. Attacks that stay inside every
coordinate-wise or distance-based spread (e.g. `alie`, `min-max`) still stretch the covariance along one direction, which SMEA sees.

  distances D = the fp32 squared distances of Krum / MDA (of the mixed or clipped rows with a pre-aggregation);
  score     per kept set S (m = n - f rows): the largest diagonal entry of B_S = -1/2 (D_ij - r_i - r_j + g) over S (DnC's double
            centring, float64) after DnC's cyclic Jacobi (same rounds, rotations, stop test and 32-sweep budget), i.e. m times the
            largest eigenvalue of the covariance of S; +inf when a distance between two members of S is not finite; 0 for m = 1;
  select    the set of smallest score (doubles, non-finite last, -0 == +0); ties -> the lexicographically smallest sorted id list;
  output    the mean of the rows of S, added in ascending worker order from +0 and divided once (Krum's selection mean).

Needs 0 <= 2 f < n and C(n, f) <= 2^14 (every f <= 7 at n <= 16, f <= 5 at n <= 20, f <= 4 at n <= 26, f <= 3 at n <= 32), which
keeps the selection under 50 ms on an H100; with f = 0 SMEA is the average.
Takes no `--aggregator-args`.

sm_90a path: the distance pass of Krum (phase A, bucketed overlap, mailbox exchange), then the C(n, f) removal sets split over the warps
of the grid, each warp running the Jacobi of its sets in a float64 slab of its own, then Krum's mean of the selected rows. Not in the
reference."""

from .. import tools
from . import _GAR, FusedSpec, register
from . import _ops


class SmeaGAR(_GAR):
  def __init__(self, nbworkers, nbbyzwrks, args):
    unknown = sorted(tools.parse_keyval(args if args is not None else []))
    if unknown:
      raise tools.UserException("SMEA takes no --aggregator-args (got %s)" % ", ".join(map(repr, unknown)))
    _ops.check_smea(nbworkers, nbbyzwrks)
    self._n, self._f = nbworkers, nbbyzwrks

  def aggregate(self, gradients):
    G = _ops.stack(gradients)
    n, f = G.shape[0], self._f
    _ops.check_smea(n, f)
    return _ops.dispatch(G, lambda M: _ops.host_smea(M, f), FusedSpec("smea", n, f=f))

  def fused_spec(self):
    return FusedSpec("smea", self._n, f=self._f)


register("smea", SmeaGAR)

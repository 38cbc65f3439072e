"""`geometric-median`: the geometric median argmin_z sum_i ||z - x_i|| (RFA, Pillutla et al., "Robust Aggregation for Federated
Learning"), approximated by smoothed Weiszfeld iterations from the coordinate-wise median:

  z_0 = the `median` rule's output (finite ascending, non-finite last, ties -> lower worker index);
  for t < T: D_i = ||z_t - x_i||^2; rows with a non-finite D_i are skipped; beta_i = 1 / max(nu, sqrt(D_i));
             z_{t+1} = (sum beta_i x_i) / (sum beta_i), both sums over the kept rows in ascending worker order from +0;
             no kept row: z_{t+1} = z_t.

fp32, every operation rounded once (no FMA): given the distances, every back-end computes the same bits. Rotation invariant,
breakdown point 1/2. `--aggregator-args iterations:<int> nu:<float>` (default 3 and 1e-6; 1 <= iterations <= 16, nu finite > 0,
rounded once to fp32). f is not used by the algorithm but must satisfy 0 <= 2f < n.

sm_90a path: T + 1 passes of the finish kernel over the owned coordinates (the median, then one pass per iteration from a
staged copy), with one cross-rank exchange of the n distances per iteration. Not in the reference."""

from .. import tools
from . import _GAR, FusedSpec, register
from . import _ops


class GeometricMedianGAR(_GAR):
  def __init__(self, nbworkers, nbbyzwrks, args):
    parsed = tools.parse_keyval(args if args is not None else [], defaults={"iterations": 3, "nu": 1e-6})
    self._iterations, self._nu = _ops.check_geometric_median(nbworkers, nbbyzwrks, parsed["iterations"], parsed["nu"])
    self._n, self._f = nbworkers, nbbyzwrks

  def _spec(self, n):
    return FusedSpec("geometric-median", n, f=self._f, iterations=self._iterations, nu=self._nu)

  def aggregate(self, gradients):
    G = _ops.stack(gradients)
    n = G.shape[0]
    _ops.check_geometric_median(n, self._f, self._iterations, self._nu)
    return _ops.dispatch(G, lambda M: _ops.host_geometric_median(M, self._iterations, self._nu), self._spec(n))

  def fused_spec(self):
    return self._spec(self._n)


register("geometric-median", GeometricMedianGAR)

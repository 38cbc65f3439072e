"""`dnc`: divide-and-conquer (DnC, Shejwalkar and Houmansadr, "Manipulating the Byzantine: Optimizing Model Poisoning Attacks and
Defenses for Federated Learning", NDSS 2021), the defence the paper proposes against its Min-Max / Min-Sum attacks (`--attack min-max`).

Every iteration t < T samples b coordinates of the flat gradient, finds the direction of largest spread of the n sampled rows and
removes the r = floor(c f) rows that stand out most along it; the output is the mean of the rows no iteration removed:

  sample   b' = min(b, D) distinct coordinates s_k = P(k) of [0, D), P a keyed permutation of step `step` and iteration t
           (`_ops.dnc_sample`: a 4-round Feistel network on splitmix64, cycle-walked; NumPy, C++ and CUDA agree bit for bit);
  distance D^t_ij = sum_k (x_i[s_k] - x_j[s_k])^2 (fp32); the rows with the most non-finite distances are dropped one at a time
           (highest index first) until every remaining distance is finite, and score +inf;
  score    s_i = u_i^2, u the top eigenvector of the double-centred Gram matrix B = -1/2 (D_ij - r_i - r_j + g) of the remaining rows
           (float64 cyclic Jacobi, every operation rounded once: the same bits on every back-end), which ranks the rows as the paper's
           <x_i - mu, v>^2 = lambda_1 u_i^2 does;
  keep     the n - r rows first under the ordering convention (finite ascending, non-finite last, ties -> lower index); the good set
           is the intersection over the T iterations;
  output   the mean of the good rows, added in ascending worker order from +0 and divided once (Krum's selection mean).

`--aggregator-args iterations:<int> subsample:<int> c:<float> seed:<int>` (default 1, 10000, 1.0 and 0; 1 <= iterations <= 8,
1 <= subsample <= 2^20, c finite >= 0, 0 <= seed < 2^64). The defaults are this project's, not values tuned in the paper. Requires
0 <= 2 f < n and n - iterations * r >= 1; with f = 0 (or c = 0) DnC is the average.

D is the row length the caller sees: the padded flat size on the aggregation engines, G's row length for a direct call. The step key is
the number of the optimizer update the aggregation feeds (checkpointed: a resumed run draws the same samples); calling `aggregate`
directly takes `step=` (an integer in [0, 2^63), on every back-end), and otherwise counts its own calls from 1.

sm_90a path: a finish kernel of its own (`gar_dnc_kernel`), with a sampled distance pass over a compact gathered copy of the sampled
coordinates, one cross-rank exchange of the T sampled distance matrices, the Jacobi in every CTA, then Krum's phase D. Not in the
reference."""

from .. import tools
from . import _GAR, FusedSpec, register
from . import _ops


class DncGAR(_GAR):
  def __init__(self, nbworkers, nbbyzwrks, args):
    parsed = tools.parse_keyval(args if args is not None else [], defaults={"iterations": 1, "subsample": 10000, "c": 1.0, "seed": 0})
    self._params = _ops.check_dnc(nbworkers, nbbyzwrks, parsed["iterations"], parsed["subsample"], parsed["c"], parsed["seed"])[:4]
    self._n, self._f = nbworkers, nbbyzwrks
    self._calls = 0

  def _spec(self, n):
    iterations, subsample, c, seed = self._params
    return FusedSpec("dnc", n, f=self._f, iterations=iterations, subsample=subsample, c=c, seed=seed)

  def aggregate(self, gradients, step=None):
    """Aggregate with step key `step`; without one, the number of calls of this object so far (this one included)."""
    G = _ops.stack(gradients)
    _ops.check_dnc(G.shape[0], self._f, *self._params)
    if step is None:
      self._calls += 1
      step = self._calls
    if G.is_cuda:
      from ..ops import gar as gar_ops
      return gar_ops.aggregate(self._spec(G.shape[0]), G, step=step)
    return _ops.host_dnc(G, self._f, *self._params, step)

  def fused_spec(self):
    return self._spec(self._n)


register("dnc", DncGAR)

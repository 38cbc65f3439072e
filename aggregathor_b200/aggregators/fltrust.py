"""`fltrust`: FLTrust (Cao, Fang, Liu and Gong, "FLTrust: Byzantine-robust Federated Learning via Trust Bootstrapping", NDSS 2021).

The parameter server holds a small clean root dataset and computes its own gradient r on it every step. Each row x_i is trusted as far
as it points the same way as r, and rescaled to r's norm:

  TS_i = ReLU(cos(x_i, r)),   x'_i = (||r|| / ||x_i||) x_i,   output = sum TS_i x'_i / sum TS_i   (+0 when sum TS_i = 0).

Unlike the statistical rules, it does not infer the honest rows from the submitted rows alone, so a colluding minority that stays
inside the honest spread (ALIE, Min-Max, Fang et al.'s attacks) does not defeat it. The exact arithmetic, shared by every back-end, is
in `_ops.py`. f is not used (any 0 <= f < n).

`--aggregator-args root-size:<m>` (default 100, the paper's): the size of the root dataset, drawn from the experiment's training set
(`experiments._Experiment.root_stream`). The trainer runs one extra forward/backward per step on a root batch, on rank 0 only, into the
engine's root row (`needs_root`). FLTrust is refused with a pre-aggregation (NNM, ARC and bucketing change the rows whose direction
and norm it scores) and with worker momentum (the rows would be momenta, the root a raw gradient).

sm_90a path: a finish kernel of its own (`gar_fltrust_kernel`): one pass for the sums (the root read from rank 0 over P2P), one
cross-rank exchange of the 2n + 1 sums, the float64 coefficients on warp 0 of every CTA, then the weighted sum, the optimizer and the
parameter broadcast. Not in the reference."""

from .. import tools
from . import _GAR, FusedSpec, register
from . import _ops


class FLTrustGAR(_GAR):
  needs_root = True

  def __init__(self, nbworkers, nbbyzwrks, args):
    parsed = tools.parse_keyval(args if args is not None else [], defaults={"root-size": _ops.FLTRUST_ROOT_SIZE})
    self.root_size = _ops.check_fltrust(nbworkers, nbbyzwrks, parsed["root-size"])
    self._n, self._f = nbworkers, nbbyzwrks

  def _spec(self, n):
    return FusedSpec("fltrust", n, f=self._f)

  def aggregate(self, gradients, root=None):
    """Aggregate against the root gradient `root` ([d], required)."""
    G = _ops.stack(gradients)
    if root is None:
      raise tools.UserException("FLTrust aggregates against a root gradient: pass root=")
    if G.is_cuda:
      from ..ops import gar as gar_ops
      return gar_ops.aggregate(self._spec(G.shape[0]), G, root=root)
    return _ops.host_fltrust(G, root)

  def fused_spec(self):
    return self._spec(self._n)


register("fltrust", FLTrustGAR)

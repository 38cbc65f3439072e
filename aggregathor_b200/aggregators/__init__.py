"""Gradient aggregation rules (GARs) — plug-in registry and base class.

Contract kept from the reference (`aggregators/__init__.py:40-70`):
`register(name, cls)`, `instantiate(name, nbworkers, nbbyzwrks, args)`,
`itemize()`; a GAR is built as `cls(nbworkers, nbbyzwrks, args)` (`args` is the
raw `key:value` list of `--aggregator-args`) and exposes
`aggregate(gradients) -> flat gradient`, where `gradients` is a list of `n`
flat 1-D tensors (or an `[n, d]` tensor). Dropping a new `.py` file in this
directory auto-registers it.

Addition: `fused_spec()` describes the rule to the fused
gather+aggregate+update kernel (`parallel/fused.py`); rules returning `None`
(e.g. user plug-ins) are run through the generic gather -> `aggregate()` ->
optimizer path.
"""

import pathlib

from .. import tools

__all__ = ["_GAR", "FusedSpec", "register", "instantiate", "itemize", "get"]


class FusedSpec:
  """What the fused sm_90a aggregation kernel needs to know about a rule."""

  RULES = ("average", "average-nan", "median", "averaged-median", "krum", "bulyan", "trimmed-mean", "mda", "geometric-median",
           "centered-clipping")

  def __init__(self, rule, n, f=0, m=0, beta=0, *, iterations=3, nu=1e-6, tau=10.0):
    """`iterations` and `nu` are the geometric median's Weiszfeld iterations and smoothing, `iterations` and `tau` centered
    clipping's iterations and clipping radius; the other rules ignore them."""
    if rule not in self.RULES:
      raise tools.UserException("Unknown fused rule " + repr(rule))
    self.rule, self.n, self.f, self.m, self.beta = rule, int(n), int(f), int(m), int(beta)
    self.iterations, self.nu, self.tau = int(iterations), float(nu), float(tau)

  @property
  def rule_id(self):
    return self.RULES.index(self.rule)

  def __repr__(self):
    extra = {"geometric-median": ", iterations=%d, nu=%r" % (self.iterations, self.nu),
             "centered-clipping": ", iterations=%d, tau=%r" % (self.iterations, self.tau)}.get(self.rule, "")
    return "FusedSpec(rule=%r, n=%d, f=%d, m=%d, beta=%d%s)" % (self.rule, self.n, self.f, self.m, self.beta, extra)


class _GAR:
  """Base gradient aggregation rule."""

  def __init__(self, nbworkers, nbbyzwrks, args):
    """`nbworkers`: total number of workers n; `nbbyzwrks`: declared Byzantine workers f; `args`: `key:value` list."""
    raise NotImplementedError

  def aggregate(self, gradients):
    """Aggregate `n` flat gradients (list of 1-D tensors or `[n, d]` tensor) into one flat gradient."""
    raise NotImplementedError

  def fused_spec(self):
    """`FusedSpec` for the fused kernel path, or None when only `aggregate()` is available."""
    return None


_register = tools.ClassRegister("GAR")
itemize = _register.itemize
register = _register.register
instantiate = _register.instantiate
get = _register.get
del _register

with tools.Context("aggregators", None):
  tools.import_directory(pathlib.Path(__file__).parent, globals())

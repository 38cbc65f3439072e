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

import math
import pathlib

from .. import tools

__all__ = ["_GAR", "FusedSpec", "register", "instantiate", "itemize", "get"]


class FusedSpec:
  """What the fused sm_90a aggregation kernel needs to know about a rule."""

  RULES = ("average", "average-nan", "median", "averaged-median", "krum", "bulyan", "trimmed-mean", "mda", "geometric-median",
           "centered-clipping", "dnc", "smea", "fltrust", "foolsgold")

  RULES_WITH_F = ("krum", "bulyan", "trimmed-mean", "mda", "geometric-median", "centered-clipping", "dnc", "smea")   # the others ignore f
  MIXES = (None, "nnm", "arc", "arc+nnm")   # the index is the kernel's bit mask: MIX_NNM | MIX_ARC
  MIX_NNM, MIX_ARC = 1, 2
  # bucketing is a mix of its own (bit MIX_BUCKETING alone, never combined with NNM or ARC), complete only with its bucket size
  BUCKETING, MIX_BUCKETING = "bucketing", 4

  def __init__(self, rule, n, f=0, m=0, beta=0, *, iterations=3, nu=1e-6, tau=10.0, mix=None, subsample=10000, c=1.0, seed=0, bucket_size=None,
               confidence=1.0):
    """`iterations` and `nu` are the geometric median's Weiszfeld iterations and smoothing, `iterations` and `tau` centered
    clipping's iterations and clipping radius, `iterations`, `subsample`, `c` and `seed` DnC's iterations, sampled coordinates,
    filtering fraction and sampling seed, `confidence` FoolsGold's kappa; the other rules ignore them. `mix` is the pre-aggregation run on the rows before the
    rule, with the same f: None, "nnm" (nearest-neighbour mixing), "arc" (adaptive robust clipping) or "arc+nnm" (ARC, then NNM on
    the clipped rows), or "bucketing" with `bucket_size` s: then `n` is the rule's row count n' = ceil(n_rows / s), the number of
    bucket means, and the kernel gathers the n_rows rows it is given."""
    if rule not in self.RULES:
      raise tools.UserException("Unknown fused rule " + repr(rule))
    if mix not in self.MIXES and mix != self.BUCKETING:
      raise tools.UserException("Unknown pre-aggregation " + repr(mix))
    if mix == self.BUCKETING and (isinstance(bucket_size, bool) or not isinstance(bucket_size, int) or bucket_size < 1):
      raise tools.UserException("Bucketing needs a bucket size s >= 1 (got %r)" % (bucket_size,))
    self.rule, self.n, self.f, self.m, self.beta = rule, int(n), int(f), int(m), int(beta)
    self.iterations, self.nu, self.tau = int(iterations), float(nu), float(tau)
    self.mix = mix
    self.bucket_size = bucket_size if mix == self.BUCKETING else None
    self.subsample, self.c, self.seed = int(subsample), float(c), int(seed)
    self.confidence = float(confidence)

  @property
  def rule_id(self):
    return self.RULES.index(self.rule)

  @property
  def mix_id(self):
    return self.MIX_BUCKETING if self.mix == self.BUCKETING else self.MIXES.index(self.mix)

  def with_mix(self, mix, f=None, bucket_size=None):
    """The same rule with pre-aggregation `mix` (one of `MIXES`, or "bucketing" with `bucket_size`), and declared f `f` (default:
    unchanged)."""
    return self.with_rows(self.n, mix=mix, f=f, bucket_size=bucket_size)

  def with_rows(self, n, mix=(), f=None, bucket_size=None):
    """The same rule for `n` rows (every other parameter unchanged unless given)."""
    mix, bucket_size = (self.mix, self.bucket_size) if mix == () else (mix, bucket_size)
    return FusedSpec(self.rule, n, self.f if f is None else f, self.m, self.beta, iterations=self.iterations, nu=self.nu, tau=self.tau,
                     mix=mix, subsample=self.subsample, c=self.c, seed=self.seed, bucket_size=bucket_size, confidence=self.confidence)

  def gathered_rows(self, n_rows):
    """Whether the rule's n rows are what `n_rows` gathered rows give: n_rows itself, or ceil(n_rows / s) with bucketing."""
    return self.n == (n_rows if self.mix != self.BUCKETING else (n_rows + self.bucket_size - 1) // self.bucket_size)

  @property
  def removed(self):
    """DnC: the rows every iteration removes, r = floor(c f) in float64."""
    return math.floor(self.c * self.f)

  def __repr__(self):
    extra = {"geometric-median": ", iterations=%d, nu=%r" % (self.iterations, self.nu),
             "centered-clipping": ", iterations=%d, tau=%r" % (self.iterations, self.tau),
             "dnc": ", iterations=%d, subsample=%d, c=%r, seed=%d" % (self.iterations, self.subsample, self.c, self.seed),
             "foolsgold": ", confidence=%r" % self.confidence}.get(self.rule, "")
    if self.mix is not None:
      extra += ", mix=%r" % self.mix
    if self.bucket_size is not None:
      extra += ", bucket_size=%d" % self.bucket_size
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

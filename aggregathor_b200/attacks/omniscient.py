"""Omniscient, colluding attacks: the Byzantine workers see the honest gradients and all send the same crafted row.

* `alie`  "A Little Is Enough" (Baruch, Baruch, Goldberg, NeurIPS 2019): b = mu + z * sigma, with the coordinate-wise mean and unbiased
          standard deviation of the honest rows. `z` defaults to z_max = Phi^-1((n - s) / n), s = floor(n / 2 + 1) - k, the largest shift
          that keeps the Byzantine rows inside the crowd the rule is supposed to trust.
* `ipm`   inner-product manipulation ("Fall of Empires", Xie, Koyejo, Gupta, UAI 2019): b = -epsilon * mu (`epsilon` defaults to 0.1).
* `min-max`, `min-sum`  the AGR-agnostic attacks of Shejwalkar & Houmansadr ("Manipulating the Byzantine: Optimizing Model Poisoning
          Attacks and Defenses for Federated Learning", NDSS 2021): b = mu - gamma * p along the deviation p (`deviation:unit-vec`, the
          default: p = mu, whose normalisation is folded into gamma; `sign`: sign(mu); `std`: ALIE's sigma), with the largest gamma that
          keeps b inside the spread of the honest rows: Min-Max bounds max_i ||b - h_i||^2 by the largest honest distance
          max_jk ||h_j - h_k||^2, Min-Sum bounds sum_i ||b - h_i||^2 by max_i sum_j ||h_i - h_j||^2. gamma is solved in closed form
          (`aggregators._ops.optimized_gamma`) instead of the authors' search, and is not capped (their search stays below 20).
* `mimic` (Karimireddy, He & Jaggi, "Byzantine-Robust Learning on Heterogeneous Datasets via Bucketing", ICLR 2022): every Byzantine
          row is a copy of one honest row h_{i*}, which over-weights that worker's data without sending any outlier. During the first
          `warmup` steps (T0, default 100) i* follows the honest row furthest along the top principal direction of the honest rows,
          estimated by an online power iteration; then i* is frozen. It does nothing under IID data and is the standard test of the
          heterogeneity defences (bucketing, NNM) under non-IID data (`dirichlet:<alpha>`). The arithmetic is
          `aggregators._ops.torch_mimic_step_`; the engine keeps the state (z, t, i*) and checkpoints it.
* `fang-krum`, `fang-trim`  the full-knowledge local model poisoning attacks of Fang, Cao, Jia & Gong ("Local Model Poisoning Attacks
          to Byzantine-Robust Federated Learning", USENIX Security 2020) against Krum and against trimmed mean (also used against median).
          The paper crafts local models w' = w - lr g'; here, as for every attack, the Byzantine rows are gradients g', so its lambda is
          gamma = lambda / lr and its direction s = -sign(mu) (mu the honest mean). Under Adam or RMSProp this gradient-space attack is
          what runs, not a model-space one.
          fang-krum: every Byzantine row is (-gamma) * sign(mu). gamma_max is the paper's upper bound on lambda in gradient units, with
          sqrt(sum p^2) in place of sqrt(d); gamma halves from gamma_max until Krum, modelled on the exchanged whole-vector sums with the
          engine's declared f, ranks a Byzantine row first, or until it falls below `threshold:<x>` (default 1e-5, in gradient units).
          All K rows are identical (the paper's other c - 1 models sit in an epsilon-ball around the first one): Krum's index-stable
          ranking then selects one of them exactly when it would select that first one (`aggregators._ops.fang_krum_gamma`).
          fang-trim: per coordinate, every Byzantine row draws its own value in the interval past the honest extreme against the sign of
          mu: [e beta, e] or [e / beta, e] below e = min_i h_i when mu > 0, [e, e beta] or [e, e / beta] above e = max_i h_i when mu < 0
          (`scale:<beta>`, the paper's b, default 2, > 1). The draw is keyed by `seed:<int>` (default 0), the update number, the row's
          slot and the coordinate, so the rows are the same bits on every engine and rank count (`aggregators._ops.torch_fang_trim_row`).

The rows are crafted by the aggregation engine (`craft_byzantine`), not per worker: on the fused engine every rank computes its owned
coordinates of every Byzantine row from the honest values it already reads for the rule, and stores them into the Byzantine rows over
NVLink (Min-Max / Min-Sum and fang-krum first exchange their whole-vector sums between the ranks). The exact arithmetic is
`aggregators._ops.torch_byzantine_row` and `torch_optimized_row`. The Byzantine workers are the last k logical workers.
"""

import math
import statistics
import struct

from .. import tools
from . import _Attack, register


def _fp32(value):
  """`value` rounded once to the nearest fp32 (overflow gives +-inf)."""
  try:
    return struct.unpack("f", struct.pack("f", value))[0]
  except OverflowError:
    return math.copysign(math.inf, value)


def default_z(nbworkers, nbbyzwrks):
  """z_max of Baruch et al. for n workers of which k are Byzantine, computed in double and rounded once to fp32."""
  s = (nbworkers // 2 + 1) - nbbyzwrks
  if s < 1:
    raise tools.UserException("alie: the default z needs k <= floor(n / 2) (got n = %d, k = %d); give 'z:<value>'" % (nbworkers, nbbyzwrks))
  return _fp32(statistics.NormalDist().inv_cdf((nbworkers - s) / nbworkers))


class _Omniscient(_Attack):
  omniscient = True
  mode = None
  deviation = None   # Min-Max / Min-Sum: "unit-vec", "sign" or "std"
  threshold = None   # fang-krum: smallest candidate gamma tested after the first
  scale = None   # fang-trim: beta
  seed = None   # fang-trim: seed of the draw
  min_honest = 1

  def __init__(self, nbworkers, nbbyzwrks, args):
    if not 1 <= nbbyzwrks < nbworkers:
      raise tools.UserException("%s needs between 1 and n - 1 Byzantine workers (got n = %d, k = %d)" % (self.mode, nbworkers, nbbyzwrks))
    if nbworkers - nbbyzwrks < self.min_honest:
      raise tools.UserException("%s needs at least %d honest workers (got n = %d, k = %d)" % (self.mode, self.min_honest, nbworkers, nbbyzwrks))
    self.args = tools.parse_keyval(args if args is not None else [])

  def _coefficient(self, key, default):
    """The fp32 value of argument `key` (or `default()` when absent), which must be finite."""
    if key not in self.args:
      return default()
    try:
      value = _fp32(float(self.args[key]))
    except ValueError:
      raise tools.UserException("%s: %r expects a number (got %r)" % (self.mode, key, self.args[key]))
    if not math.isfinite(value):
      raise tools.UserException("%s: %r must be finite in fp32 (got %r)" % (self.mode, key, self.args[key]))
    return value


class AlieAttack(_Omniscient):
  mode = "alie"
  min_honest = 2

  def __init__(self, nbworkers, nbbyzwrks, args):
    super().__init__(nbworkers, nbbyzwrks, args)
    self.coef = self._coefficient("z", lambda: default_z(nbworkers, nbbyzwrks))


class IpmAttack(_Omniscient):
  mode = "ipm"

  def __init__(self, nbworkers, nbbyzwrks, args):
    super().__init__(nbworkers, nbbyzwrks, args)
    self.coef = self._coefficient("epsilon", lambda: _fp32(0.1))


class _OptimizedAttack(_Omniscient):
  """Min-Max / Min-Sum: no coefficient (gamma is solved every step from the honest rows), only the deviation."""
  min_honest = 2

  def __init__(self, nbworkers, nbbyzwrks, args):
    super().__init__(nbworkers, nbbyzwrks, args)
    from ..aggregators import _ops
    unknown = set(self.args) - {"deviation"}
    if unknown:
      raise tools.UserException("%s: unknown argument(s) %s (expected 'deviation:unit-vec|sign|std')" % (self.mode, ", ".join(sorted(unknown))))
    self.deviation = _ops.check_deviation(self.mode, self.args.get("deviation"))
    self.coef = None


class MinMaxAttack(_OptimizedAttack):
  mode = "min-max"


class MinSumAttack(_OptimizedAttack):
  mode = "min-sum"


class MimicAttack(_Omniscient):
  """Mimic: no coefficient, only the warm-up length T0 (`warmup:<T0>`, an integer >= 1)."""
  mode = "mimic"
  min_honest = 2

  def __init__(self, nbworkers, nbbyzwrks, args):
    super().__init__(nbworkers, nbbyzwrks, args)
    from ..aggregators import _ops
    unknown = set(self.args) - {"warmup"}
    if unknown:
      raise tools.UserException("mimic: unknown argument(s) %s (expected 'warmup:<steps>')" % ", ".join(sorted(unknown)))
    warmup = _ops.MIMIC_WARMUP
    if "warmup" in self.args:
      try:
        warmup = int(self.args["warmup"])
      except ValueError:
        raise tools.UserException("mimic: 'warmup' expects an integer >= 1 (got %r)" % (self.args["warmup"],))
    self.warmup = _ops.check_mimic(nbworkers, range(nbworkers - nbbyzwrks, nbworkers), warmup)[1]
    self.coef = None


class FangKrumAttack(_Omniscient):
  """fang-krum: no coefficient (gamma is searched every step), only the threshold (`threshold:<x>`, finite, > 0, in gradient units)."""
  mode = "fang-krum"
  min_honest = 2

  def __init__(self, nbworkers, nbbyzwrks, args):
    super().__init__(nbworkers, nbbyzwrks, args)
    from ..aggregators import _ops
    unknown = set(self.args) - {"threshold"}
    if unknown:
      raise tools.UserException("fang-krum: unknown argument(s) %s (expected 'threshold:<x>')" % ", ".join(sorted(unknown)))
    if 2 * nbbyzwrks + 1 >= nbworkers:
      raise tools.UserException("fang-krum needs n - 2 k - 1 >= 1 (got n = %d, k = %d)" % (nbworkers, nbbyzwrks))
    self.threshold = self._coefficient("threshold", lambda: _ops.fp32(_ops.FANG_THRESHOLD))
    if not self.threshold > 0:
      raise tools.UserException("fang-krum: the threshold must be > 0 (got %r)" % (self.args["threshold"],))
    self.coef = None


class FangTrimAttack(_Omniscient):
  """fang-trim: no coefficient, the scale beta (`scale:<beta>`, finite, > 1) and the seed of the draw (`seed:<int>`, in [0, 2^64))."""
  mode = "fang-trim"

  def __init__(self, nbworkers, nbbyzwrks, args):
    super().__init__(nbworkers, nbbyzwrks, args)
    from ..aggregators import _ops
    unknown = set(self.args) - {"scale", "seed"}
    if unknown:
      raise tools.UserException("fang-trim: unknown argument(s) %s (expected 'scale:<beta>', 'seed:<int>')" % ", ".join(sorted(unknown)))
    self.scale = _ops.check_fang_scale(self._coefficient("scale", lambda: _ops.FANG_SCALE))
    seed = 0
    if "seed" in self.args:
      try:
        seed = int(self.args["seed"])
      except ValueError:
        raise tools.UserException("fang-trim: 'seed' expects an integer in [0, 2^64) (got %r)" % (self.args["seed"],))
    _ops.fang_trim_key(seed, 0)
    self.seed = seed
    self.coef = None


register("alie", AlieAttack)
register("ipm", IpmAttack)
register("min-max", MinMaxAttack)
register("min-sum", MinSumAttack)
register("mimic", MimicAttack)
register("fang-krum", FangKrumAttack)
register("fang-trim", FangTrimAttack)

"""Omniscient, colluding attacks: the Byzantine workers see the honest gradients and all send the same crafted row.

* `alie`  "A Little Is Enough" (Baruch, Baruch, Goldberg, NeurIPS 2019): b = mu + z * sigma, with the coordinate-wise mean and unbiased
          standard deviation of the honest rows. `z` defaults to z_max = Phi^-1((n - s) / n), s = floor(n / 2 + 1) - k, the largest shift
          that keeps the Byzantine rows inside the crowd the rule is supposed to trust.
* `ipm`   inner-product manipulation ("Fall of Empires", Xie, Koyejo, Gupta, UAI 2019): b = -epsilon * mu (`epsilon` defaults to 0.1).

The rows are crafted by the aggregation engine (`craft_byzantine`), not per worker: on the fused engine every rank computes its owned
coordinates of every Byzantine row from the honest values it already reads for the rule, and stores them into the Byzantine rows over
NVLink. The exact arithmetic is `aggregators._ops.torch_byzantine_row`. The Byzantine workers are the last k logical workers.
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


register("alie", AlieAttack)
register("ipm", IpmAttack)

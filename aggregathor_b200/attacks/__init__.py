"""Byzantine attacks — plug-in registry (fills the reference's `--attack` TODO, `runner.py:345`).

The reference parses `--attack/--attack-args` but never uses them; `--nb-real-byz-workers k` merely leaves k workers
uninstantiated. Here the last k logical workers are *real* Byzantine workers: they compute an honest gradient (so
that omniscient-free attacks such as sign flipping have something to transform) and the selected attack then
overwrites their row of the gradient matrix, on the device, before the aggregation kernel's entry barrier.

Contract: `cls(nbworkers, nbbyzwrks, args)`; `apply(row, worker, step, state)` mutates the flat fp32 gradient `row`
in place (`state` is a per-worker dict that persists across steps). Dropping a `.py` file here auto-registers it.
Omniscient attacks (`omniscient = True`, `omniscient.py`) see every honest row instead: they implement no `apply`, and expose `mode`
("alie" or "ipm") and the fp32 coefficient `coef`; the aggregation engine crafts the Byzantine rows (`craft_byzantine`) on every rank.
Construction raises `UserException` for arguments outside an attack's bounds.
"""

import pathlib

from .. import tools

__all__ = ["_Attack", "register", "instantiate", "itemize"]


class _Attack:
  forges = False  # True: the attack tampers with the row *after* it was signed (only meaningful with `--authenticate`)
  omniscient = False  # True: the rows are crafted from the honest rows by the aggregation engine (no `apply`)

  def __init__(self, nbworkers, nbbyzwrks, args):
    raise NotImplementedError

  def apply(self, row, worker, step, state):
    raise NotImplementedError


_register = tools.ClassRegister("attack")
itemize = _register.itemize
register = _register.register
instantiate = _register.instantiate
del _register

with tools.Context("attacks", None):
  tools.import_directory(pathlib.Path(__file__).parent, globals())

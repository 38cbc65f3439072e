"""Byzantine attacks — plug-in registry (fills the reference's `--attack` TODO, `runner.py:345`).

The reference parses `--attack/--attack-args` but never uses them; `--nb-real-byz-workers k` merely leaves k workers
uninstantiated. Here the last k logical workers are *real* Byzantine workers: they compute an honest gradient (so
that omniscient-free attacks such as sign flipping have something to transform) and the selected attack then
overwrites their row of the gradient matrix, on the device, before the aggregation kernel's entry barrier.

Contract: `cls(nbworkers, nbbyzwrks, args)`; `apply(row, worker, step, state)` mutates the flat fp32 gradient `row`
in place (`state` is a per-worker dict that persists across steps). Dropping a `.py` file here auto-registers it.
Omniscient attacks (`omniscient = True`, `omniscient.py`) see every honest row instead: they implement no `apply`, and expose `mode`
("alie", "ipm", "min-max", "min-sum", "mimic", "fang-krum" or "fang-trim"), the fp32 coefficient `coef` (None for Min-Max / Min-Sum and
fang-krum, which solve theirs every step, and for mimic and fang-trim), `deviation` (Min-Max / Min-Sum; None otherwise), `warmup` (mimic
only), `threshold` (fang-krum only), `scale` and `seed` (fang-trim only); the aggregation engine crafts the Byzantine rows
(`craft_byzantine`) on every rank.
Data-poisoning attacks (`poisons_data = True`, `data.py`) implement no `apply` either: the Byzantine workers train on poisoned data, so
nothing rewrites their rows after the backward pass. Label flipping (`flips_labels = True`) has their loss train on flipped labels (the
trainer sets `Context.flip_from`); the backdoor exposes `target`, `fraction`, `scale`, `poisoned_rows(batch_size)` and
`check_target(classes)`, and the trainer sets `Context.backdoor` from them.
Construction raises `UserException` for arguments outside an attack's bounds.
"""

import pathlib

from .. import tools

__all__ = ["_Attack", "register", "instantiate", "itemize"]


class _Attack:
  forges = False  # True: the attack tampers with the row *after* it was signed (only meaningful with `--authenticate`)
  omniscient = False  # True: the rows are crafted from the honest rows by the aggregation engine (no `apply`)
  poisons_data = False  # True: the Byzantine workers compute their gradient on poisoned data (no `apply`)
  flips_labels = False  # True: the data poisoning is label flipping

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

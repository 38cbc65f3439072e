"""The host checks of the five crafting entry points of `op_gar`: every invalid argument block is refused with its status, before
anything is launched, and an argument block that fails two checks gets the status of the check that comes first."""

import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

N, D = 6, 64
HONEST, BYZ = 0b111110, 0b000001   # slot 0 Byzantine, slots 1-5 honest
ALIE, IPM, MIN_MAX, MIN_SUM = 0, 1, 2, 3
UNIT_VEC, STD = 0, 2


class _Env:
  def __init__(self):
    from aggregathor_b200.ops import gar as gar_ops
    self.lib = gar_ops._lib()
    for name in ("agb_gar_byzantine", "agb_gar_byzantine_optimized", "agb_gar_byzantine_mimic", "agb_gar_byzantine_fang_krum",
                 "agb_gar_byzantine_fang_trim"):
      getattr(self.lib, name).restype = ctypes.c_int
    self.stream = gar_ops._stream_ptr()
    # real buffers behind every address, although none of these calls may reach a kernel
    self.G = torch.zeros((N, D), device="cuda")
    self.signal = torch.zeros(2, 1 << 12, dtype=torch.int32, device="cuda")
    self.mailbox = torch.zeros(2, 1 << 16, device="cuda")
    self.partials = torch.zeros(1 << 16, device="cuda")
    self.stats = torch.zeros(1 << 10, dtype=torch.float64, device="cuda")
    self.z, self.y = torch.zeros(D, device="cuda"), torch.zeros(D, device="cuda")
    self.istar = torch.zeros(1, dtype=torch.int32, device="cuda")

  def rows(self, n):
    return (ctypes.c_ulonglong * n)(*[self.G.data_ptr() + (i % N) * D * 4 for i in range(n)])

  def signals(self, R, present=True):
    """R signal pad addresses; `present` False: none at all, a list: which of them are set."""
    if present is False:
      return None
    present = [True] * R if present is True else present
    return (ctypes.c_ulonglong * R)(*[self.signal[q % 2].data_ptr() if present[q] else 0 for q in range(R)])

  def mailboxes(self, R, present=True):
    if present is False:
      return None
    present = [True] * R if present is True else present
    return (ctypes.c_ulonglong * R)(*[self.mailbox[q % 2].data_ptr() if present[q] else 0 for q in range(R)])

  def common(self, n=N, lo=(0,), hi=(D,), nseg=None, honest=HONEST, byzantine=BYZ):
    size = max(len(lo), nseg or 0, 1)
    seg_lo = (ctypes.c_longlong * size)(*lo)
    seg_hi = (ctypes.c_longlong * size)(*hi)
    return (self.rows(n), ctypes.c_int(n), seg_lo, seg_hi, ctypes.c_int(len(lo) if nseg is None else nseg), ctypes.c_uint(honest),
            ctypes.c_uint(byzantine))

  def byzantine(self, mode=ALIE, coef=1.0, R=1, rank=0, signals=True, **common):
    return self.lib.agb_gar_byzantine(*self.common(**common), ctypes.c_int(mode), ctypes.c_float(coef), ctypes.c_int(R), ctypes.c_int(rank),
                                      self.signals(R, signals), ctypes.c_uint(1), ctypes.c_ulonglong(0), self.stream)

  def optimized(self, mode=MIN_MAX, deviation=UNIT_VEC, R=1, rank=0, signals=True, mailboxes=True, partials=True, partial_ctas=4, **common):
    return self.lib.agb_gar_byzantine_optimized(
      *self.common(**common), ctypes.c_int(mode), ctypes.c_int(deviation), ctypes.c_int(R), ctypes.c_int(rank), self.signals(R, signals),
      self.mailboxes(R, mailboxes), ctypes.c_ulonglong(self.partials.data_ptr() if partials else 0), ctypes.c_int(partial_ctas),
      ctypes.c_ulonglong(self.stats.data_ptr()), ctypes.c_uint(1), ctypes.c_ulonglong(0), self.stream)

  def mimic(self, warmup=1, t=0, R=1, rank=0, signals=True, mailboxes=True, partials=True, partial_ctas=4, z=True, y=True, istar=True,
            **common):
    addr = lambda t, present: ctypes.c_ulonglong(t.data_ptr() if present else 0)
    return self.lib.agb_gar_byzantine_mimic(
      *self.common(**common), ctypes.c_int(warmup), ctypes.c_int(t), ctypes.c_int(R), ctypes.c_int(rank), self.signals(R, signals),
      self.mailboxes(R, mailboxes), addr(self.partials, partials), ctypes.c_int(partial_ctas), addr(self.z, z), addr(self.y, y),
      addr(self.istar, istar), ctypes.c_ulonglong(self.stats.data_ptr()), ctypes.c_uint(1), ctypes.c_ulonglong(0), self.stream)

  def fang_krum(self, f=1, threshold=1e-5, R=1, rank=0, signals=True, mailboxes=True, partials=True, partial_ctas=4, **common):
    return self.lib.agb_gar_byzantine_fang_krum(
      *self.common(**common), ctypes.c_int(f), ctypes.c_float(threshold), ctypes.c_int(1), ctypes.c_int(R), ctypes.c_int(rank),
      self.signals(R, signals), self.mailboxes(R, mailboxes), ctypes.c_ulonglong(self.partials.data_ptr() if partials else 0),
      ctypes.c_int(partial_ctas), ctypes.c_ulonglong(self.stats.data_ptr()), ctypes.c_ulonglong(self.stats.data_ptr()), ctypes.c_uint(1),
      ctypes.c_ulonglong(0), self.stream)

  def fang_trim(self, scale=2.0, R=1, rank=0, signals=True, **common):
    return self.lib.agb_gar_byzantine_fang_trim(*self.common(**common), ctypes.c_float(scale), ctypes.c_ulonglong(7), ctypes.c_int(R),
                                                ctypes.c_int(rank), self.signals(R, signals), ctypes.c_uint(1), ctypes.c_ulonglong(0),
                                                self.stream)


@pytest.fixture(scope="module")
def env():
  return _Env()


# the checks every entry point makes, in their order: workers, ranks and rank (100), segment count (101), slot masks (114), segment
# bounds (101), signal pads (109)
COMMON = [
  (dict(n=0), 100), (dict(n=33), 100), (dict(R=0), 100), (dict(R=17), 100), (dict(R=2, rank=2), 100), (dict(rank=-1), 100),
  (dict(nseg=0), 101), (dict(nseg=9), 101),
  (dict(honest=HONEST | BYZ), 114), (dict(byzantine=0), 114), (dict(honest=HONEST | 1 << N), 114), (dict(byzantine=BYZ | 1 << 31), 114),
  (dict(lo=(2,)), 101), (dict(hi=(D - 1,)), 101), (dict(lo=(8,), hi=(4,)), 101), (dict(lo=(0, 32), hi=(32, 30)), 101),
  (dict(R=2, signals=False), 109), (dict(R=2, signals=[True, False]), 109),
  # two failures: the first check decides
  (dict(n=0, nseg=0), 100), (dict(nseg=0, byzantine=0), 101), (dict(byzantine=0, lo=(2,)), 114), (dict(lo=(2,), R=2, signals=False), 101),
]


@pytest.mark.parametrize("entry", ["byzantine", "optimized", "mimic", "fang_krum", "fang_trim"])
def test_common_checks(env, entry):
  for args, status in COMMON:
    assert getattr(env, entry)(**args) == status, (entry, args)


def test_byzantine_checks(env):
  assert env.byzantine(honest=0b000010, byzantine=0b111101) == 114   # ALIE needs H >= 2
  assert env.byzantine(mode=IPM, honest=0b000010, byzantine=0b111101, lo=(0,), hi=(0,)) == 0   # IPM: H >= 1; nothing owned, no launch
  assert env.byzantine(mode=IPM, honest=0, byzantine=0b111111) == 114
  assert env.byzantine(mode=MIN_MAX) == 114 and env.byzantine(mode=-1) == 114
  assert env.byzantine(mode=MIN_MAX, nseg=0) == 101
  assert env.byzantine(mode=MIN_MAX, lo=(2,)) == 114


def test_optimized_checks(env):
  assert env.optimized(mode=ALIE) == 118 and env.optimized(mode=MIN_SUM, deviation=STD + 1) == 118
  assert env.optimized(deviation=-1) == 118
  assert env.optimized(honest=0b000010, byzantine=0b111101) == 114   # H >= 2
  assert env.optimized(mode=ALIE, honest=HONEST | BYZ) == 118   # 118 before 114
  assert env.optimized(mode=ALIE, nseg=0) == 101 and env.optimized(mode=ALIE, n=0) == 100
  assert env.optimized(mailboxes=False) == 108 and env.optimized(R=2, mailboxes=[True, False]) == 108
  assert env.optimized(partials=False) == 108 and env.optimized(partial_ctas=0) == 108
  # signal pads and mailboxes are checked rank by rank
  assert env.optimized(R=2, signals=[True, False], mailboxes=[False, True]) == 108
  assert env.optimized(R=2, signals=[False, True], mailboxes=[True, False]) == 109
  assert env.optimized(lo=(2,), mailboxes=False) == 101 and env.optimized(mailboxes=False, partials=False) == 108


def test_mimic_checks(env):
  assert env.mimic(honest=0b000010, byzantine=0b111101) == 124   # H >= 2, after the slot masks
  assert env.mimic(honest=0, byzantine=0b111111) == 124
  assert env.mimic(warmup=2) == 124 and env.mimic(t=-1) == 124 and env.mimic(t=1 << 24) == 124
  assert env.mimic(istar=False) == 124 and env.mimic(istar=False, warmup=0) == 124
  assert env.mimic(z=False) == 124 and env.mimic(y=False) == 124
  assert env.mimic(istar=False, byzantine=0) == 114   # 114 before 124
  assert env.mimic(istar=False, lo=(2,)) == 124   # 124 before the segment bounds
  assert env.mimic(istar=False, nseg=0) == 101
  assert env.mimic(mailboxes=False) == 108 and env.mimic(R=2, mailboxes=[True, False]) == 108
  assert env.mimic(partials=False) == 108 and env.mimic(partial_ctas=0) == 108
  assert env.mimic(R=2, signals=[True, False], mailboxes=[False, True]) == 108
  assert env.mimic(R=2, signals=[False, True], mailboxes=[True, False]) == 109
  assert env.mimic(warmup=0, R=2, signals=[True, False], mailboxes=False) == 109   # the copy pass needs no mailbox
  assert env.mimic(warmup=0, lo=(0,), hi=(0,), mailboxes=False, partials=False, z=False, y=False) == 0   # nothing owned, no launch


def test_fang_krum_checks(env):
  assert env.fang_krum(honest=0b011110) == 125   # every row honest or Byzantine
  assert env.fang_krum(f=-1) == 125 and env.fang_krum(f=4) == 125   # n - f - 2 >= 1
  assert env.fang_krum(honest=0b111000, byzantine=0b000111) == 125   # n - 2 K - 1 >= 1
  assert env.fang_krum(honest=0b100000, byzantine=0b011111) == 125
  assert env.fang_krum(honest=0, byzantine=0b111111) == 114   # H >= 1 under the slot masks
  assert env.fang_krum(threshold=0.0) == 125 and env.fang_krum(threshold=float("inf")) == 125 and env.fang_krum(threshold=float("nan")) == 125
  assert env.fang_krum(threshold=0.0, lo=(2,)) == 101 and env.fang_krum(threshold=0.0, R=2, signals=False) == 109
  assert env.fang_krum(mailboxes=False) == 108 and env.fang_krum(R=2, mailboxes=[True, False]) == 108
  assert env.fang_krum(threshold=0.0, mailboxes=False) == 125   # 125 before 108
  assert env.fang_krum(R=2, signals=[True, False], mailboxes=False) == 109   # the signal pads before the mailboxes
  assert env.fang_krum(partials=False) == 108 and env.fang_krum(partial_ctas=0) == 108


def test_fang_trim_checks(env):
  assert env.fang_trim(scale=1.0) == 125 and env.fang_trim(scale=float("inf")) == 125 and env.fang_trim(scale=float("nan")) == 125
  assert env.fang_trim(honest=0, byzantine=0b111111) == 114
  assert env.fang_trim(scale=1.0, lo=(2,)) == 101 and env.fang_trim(scale=1.0, R=2, signals=False) == 109
  assert env.fang_trim(scale=1.0, byzantine=0) == 114
  assert env.fang_trim(honest=0b000010, byzantine=0b111101, lo=(0,), hi=(0,)) == 0   # H = 1 is enough; nothing owned, no launch

"""Python front-end of the sm_90a aggregation kernels (`native/op_gar`).

`aggregate(spec, G)` is the stand-alone `[n, d] -> [d]` custom op (the `-co` flavour of
the reference, which only ever had a CPU kernel: `native/op_krum/op.cpp:98-107`).
`FusedLauncher` drives the full gather + rule + optimizer + broadcast kernel for one rank
(see `parallel/fused.py` for the multi-GPU wiring).
"""

import ctypes
import functools
import os

import torch

from .. import tools
from ..aggregators import FusedSpec
from . import counters

MAX_WORKERS = 32
MAX_RANKS = 16
MAX_PAIRS = MAX_WORKERS * (MAX_WORKERS - 1) // 2
MAX_SEGMENTS = 8
MAX_ITERATIONS = 16   # geometric median, centered clipping: iterations
# Min-Max / Min-Sum statistics of one rank: honest pair distances [0, 496), A_i [496, 528), B_i [528, 560), C [560]; mimic posts into the
# same region: s_i [0, 32) in its first exchange, q_i [32, 64) and ||y||^2 [64] in its second
CRAFT_STATS = MAX_PAIRS + 2 * MAX_WORKERS + 1
# mimic's statistics of a warm-up step (float64): s_i [0, 32), q_i [32, 64), ||y||^2 [64], 1 / ||y|| [65]
MIMIC_STATS = 2 * MAX_WORKERS + 2
DNC_MAX_ITERATIONS = 8
# FoolsGold's sums P_ij, i <= j, row-major upper triangle [0, n (n + 1) / 2)
FOOLSGOLD_SUMS = MAX_WORKERS * (MAX_WORKERS + 1) // 2
# FLTrust's sums and coefficients of the last launch: P [0, 32), N [32, 64), N0 [64], a [65, 97)
FLTRUST_OUT = 3 * MAX_WORKERS + 1
# FoolsGold's of the last launch: the sums [0, n (n + 1) / 2), the bad-row flags [528, 560), c [560, 592)
FOOLSGOLD_OUT = FOOLSGOLD_SUMS + 2 * MAX_WORKERS
# [0]: theta, [1, 1 + theta): selection masks; [32, 34): SMEA's winning score (float64 bits); [64, 64 + n): NNM masks;
# [96, 96 + T): DnC's mask of every iteration; bucketing: [128, 128 + n_rows) the permutation, [160, 160 + n') the bucket masks
INFO_INTS = 192
OPTIMIZERS = {"none": 0, "sgd": 1, "adam": 2, "rmsprop": 3, "adagrad": 4, "adadelta": 5}

_ERRORS = {
  100: "unsupported number of workers/ranks (n <= 32, R <= 16)", 101: "segment bounds must be multiples of 4 elements (at most 8 segments)",
  102: "unknown rule", 103: "invalid Krum parameters", 104: "invalid Bulyan parameters", 105: "invalid beta",
  106: "optimizer requested without parameter buffers", 107: "optimizer slots missing", 108: "scratch buffers missing",
  109: "signal pads missing", 110: "more than 8 workers over several ranks need the staging buffer", 111: "invalid phase A launch",
  112: "invalid trimmed-mean parameters (0 <= 2 f < n)", 113: "invalid MDA parameters (0 <= 2 f < n and C(n, f) <= 2^20)",
  114: "invalid Byzantine crafting parameters (disjoint slot masks, at least one Byzantine slot, H >= 2 for ALIE, H >= 1 for IPM)",
  115: "invalid geometric-median parameters (0 <= 2 f < n, 1 <= iterations <= 16, finite nu > 0)",
  116: "invalid centered-clipping parameters (0 <= 2 f < n, 1 <= iterations <= 16, finite tau > 0, a center buffer)",
  117: "invalid NNM parameters (0 <= 2 f < n)",
  118: "unknown Min-Max / Min-Sum mode or deviation (modes: min-max, min-sum; deviations: unit-vec, sign, std)",
  119: "invalid DnC parameters (0 <= 2 f < n, 1 <= iterations <= 8, n - iterations * r >= 1, 1 <= subsample <= 2^20, 1 <= domain <= 2^48, step >= 0)",
  120: "invalid ARC parameters (0 <= 2 f < n)", 122: "invalid SMEA parameters (0 <= 2 f < n and C(n, f) <= 2^14)",
  123: "invalid bucketing parameters (1 <= s <= n_rows, n = ceil(n_rows / s), not combined with NNM or ARC, a staging tile)",
  124: "invalid mimic parameters (H >= 2, 0 <= t < 2^24, a target buffer, and z and y buffers for a warm-up step)",
  125: "invalid Fang attack parameters (fang-krum: every row honest or Byzantine, n - f - 2 >= 1, n - 2 K - 1 >= 1, H >= 2, a finite "
       "threshold > 0; fang-trim: a finite scale > 1)",
  126: "invalid FLTrust parameters (0 <= f < n, a root gradient, no pre-aggregation, nothing pre-accumulated)",
  127: "invalid FoolsGold parameters (0 <= f < n, a finite confidence > 0, a history buffer)",
  128: "FoolsGold takes no pre-aggregation (NNM, ARC and bucketing do not keep one row per worker)",
  129: "FoolsGold runs its history pass in the finish kernel: no bucketed phase A, nothing pre-accumulated"}
ITERATIVE_RULES = ("geometric-median", "centered-clipping")   # [iterations, n] row distances in `geo_dist_out`
BYZANTINE_MODES = {"alie": 0, "ipm": 1, "min-max": 2, "min-sum": 3, "mimic": 4, "fang-krum": 5, "fang-trim": 6}
FANG_OUT = 3   # fang-krum's float64 details of the last run: gamma_max, t, selected
DEVIATIONS = {"unit-vec": 0, "sign": 1, "std": 2}


def _lib():
  from .. import native
  return native.library("op_gar")


def _stream_ptr(stream=None):
  stream = torch.cuda.current_stream() if stream is None else stream
  return ctypes.c_void_p(stream.cuda_stream)


def _check(status, what):
  counters.bump()
  if status != 0:
    raise RuntimeError("native op " + what + " failed with status " + str(status) + (" (" + _ERRORS[status] + ")" if status in _ERRORS else " (CUDA error)"))


def max_ctas():
  return int(_lib().agb_gar_max_ctas())


@functools.lru_cache(maxsize=None)
def region_bytes():
  """(signal pad, mailbox) bytes of one rank's communication regions, as the kernels lay them out."""
  out = (ctypes.c_longlong * 2)()
  _lib().agb_gar_region_bytes(out)
  return int(out[0]), int(out[1])


_ADDR = ctypes.c_ulonglong   # a pointer field of `GarArgs`: any integer address


class GarArgs(ctypes.Structure):
  """The arguments of the fused entry points: a field-for-field mirror of `struct GarArgs` in `native/op_gar/gar.cu` (see there for
  what each field means). Every pointer is a device address (`_ADDR`), 0 when absent."""
  _fields_ = [
    ("n", ctypes.c_int), ("f", ctypes.c_int), ("m", ctypes.c_int), ("beta", ctypes.c_int), ("rule", ctypes.c_int),
    ("n_rows", ctypes.c_int), ("bkt_size", ctypes.c_int), ("bkt_seed", ctypes.c_ulonglong), ("R", ctypes.c_int), ("rank", ctypes.c_int),
    ("nseg", ctypes.c_int), ("first_seg", ctypes.c_int), ("seg_lo", ctypes.c_longlong * MAX_SEGMENTS),
    ("seg_hi", ctypes.c_longlong * MAX_SEGMENTS), ("seg_ctas", ctypes.c_int * MAX_SEGMENTS), ("seg_max_ctas", ctypes.c_int),
    ("grad", _ADDR * MAX_WORKERS), ("grad_mc", _ADDR), ("workers_per_rank", ctypes.c_int),
    ("row_stride", ctypes.c_longlong), ("agg_out", _ADDR), ("opt", ctypes.c_int), ("lr", ctypes.c_float), ("h0", ctypes.c_float),
    ("h1", ctypes.c_float), ("h2", ctypes.c_float), ("hyper_ptr", _ADDR), ("param", _ADDR), ("slot0", _ADDR),
    ("slot1", _ADDR), ("param_dst", _ADDR * MAX_RANKS), ("param_mc", _ADDR),
    ("param_bf16_dst", _ADDR * MAX_RANKS), ("signal", _ADDR * MAX_RANKS), ("mailbox", _ADDR * MAX_RANKS),
    ("epoch", ctypes.c_uint32), ("epoch_ptr", _ADDR), ("cta_partials", _ADDR), ("seg_partials", _ADDR),
    ("staging", _ADDR), ("dist_out", _ADDR), ("raw_dist_out", _ADDR), ("info", _ADDR),
    ("loss_in", _ADDR), ("nloss", ctypes.c_int), ("loss_out", _ADDR), ("iterations", ctypes.c_int),
    ("nu", ctypes.c_float), ("tau", ctypes.c_float), ("center", _ADDR), ("mix", ctypes.c_int), ("arc_out", _ADDR),
    ("dnc_r", ctypes.c_int), ("dnc_b", ctypes.c_longlong), ("dnc_domain", ctypes.c_longlong), ("dnc_seed", ctypes.c_ulonglong),
    ("dnc_step", ctypes.c_longlong), ("dnc_step_ptr", _ADDR), ("dnc_scratch", _ADDR), ("smea_scratch", _ADDR),
    ("root", _ADDR), ("fltrust_out", _ADDR), ("history", _ADDR), ("foolsgold_out", _ADDR),
    ("confidence", ctypes.c_double)]


class FusedLauncher:
  """Holds the scratch buffers of one rank's fused aggregation kernels (phase A kernels + finish kernel) and fills their `GarArgs`."""

  def __init__(self, device, n, phase_a_ctas=132, phase_a_threads=128):
    if n > MAX_WORKERS:
      raise tools.UserException("The sm_90a aggregation kernels support n <= %d workers (got %d)" % (MAX_WORKERS, n))
    self.device = torch.device(device)
    self.n = n
    with torch.cuda.device(self.device):
      ctas = max(1, max_ctas())
    self.phase_a_ctas = max(1, min(int(os.environ.get("AGB_PHASE_A_CTAS", phase_a_ctas)), ctas))
    self.phase_a_threads = int(os.environ.get("AGB_PHASE_A_THREADS", phase_a_threads))
    self.cta_partials = torch.zeros(ctas * MAX_PAIRS, dtype=torch.float32, device=self.device)
    self.seg_partials = torch.zeros(MAX_SEGMENTS * self.phase_a_ctas * MAX_PAIRS, dtype=torch.float32, device=self.device)
    self.local_mailbox = torch.zeros(region_bytes()[1] // 4, dtype=torch.float32, device=self.device)
    self.dist_out = torch.zeros(n * n, dtype=torch.float32, device=self.device)
    self.geo_dist_out = torch.zeros(MAX_ITERATIONS * n, dtype=torch.float32, device=self.device)   # iterative rules: D of every iteration, [T, n]
    self.raw_dist_out = torch.zeros(n * n, dtype=torch.float32, device=self.device)   # NNM: distances of the raw rows
    self.arc_out = torch.zeros(2 * n, dtype=torch.float32, device=self.device)   # ARC: squared norms N [n], then factors c [n]
    self.dnc_dist_out = torch.zeros(DNC_MAX_ITERATIONS * n * n, dtype=torch.float32, device=self.device)   # DnC: [T, n, n] sampled distances
    self.ctas = ctas
    self._dnc_scratch = None
    self._smea_scratch = None
    self.info = torch.zeros(INFO_INTS, dtype=torch.int32, device=self.device)
    # Min-Max / Min-Sum: CTA partials of the statistics pass, and gamma followed by the statistics summed over the ranks
    self.craft_ctas = ctas
    self.craft_partials = torch.zeros(ctas * CRAFT_STATS, dtype=torch.float32, device=self.device)
    self.craft_stats = torch.zeros(1 + CRAFT_STATS, dtype=torch.float32, device=self.device)
    # mimic: the statistics of the last warm-up step, and the y scratch of the owned coordinates (`mimic_scratch`)
    self.mimic_stats = torch.zeros(MIMIC_STATS, dtype=torch.float64, device=self.device)
    self.fang_out = torch.zeros(FANG_OUT, dtype=torch.float64, device=self.device)   # fang-krum: gamma_max, t, selected
    self.fltrust_out = torch.zeros(FLTRUST_OUT, dtype=torch.float32, device=self.device)   # FLTrust: P, N, N0, a
    self.foolsgold_out = torch.zeros(FOOLSGOLD_OUT, dtype=torch.float32, device=self.device)   # FoolsGold: P, bad, c
    self._mimic_y = None
    self._func = _lib().agb_gar_fused
    self._func.argtypes = [ctypes.POINTER(GarArgs), ctypes.c_int, ctypes.c_longlong, ctypes.c_void_p]
    self._func.restype = ctypes.c_int
    self._phase_a = _lib().agb_gar_phase_a
    self._phase_a.argtypes = [ctypes.POINTER(GarArgs), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    self._phase_a.restype = ctypes.c_int
    timeout = os.environ.get("AGB_FLAG_TIMEOUT_S")
    if timeout is not None:   # bound of the cross-GPU flag waits (default 120 s, 0 = wait forever)
      with torch.cuda.device(self.device):
        _check(_lib().agb_gar_set_flag_timeout(ctypes.c_double(float(timeout))), "gar_set_flag_timeout")

  def _fill(self, spec, rows, segments, *, agg_out=None, opt="none", lr=0.0, hyper=(0.0, 0.0, 0.0), param=None, slot0=None, slot1=None, param_dst=None, param_mc=0,
            param_bf16_dst=None, rank=0, R=1, signals=None, mailboxes=None, epoch=1, staging=None, grad_mc=0, workers_per_rank=1, row_stride=0,
            first_seg=0, epoch_ptr=None, hyper_ptr=None, loss_in=None, loss_out=None, center=None, step=0, step_ptr=None, domain=None,
            bucketing_seed=0, root=None, history=None):
    """A fresh `GarArgs` of one launch (every entry it does not set is 0), and the element count of the rule's scratch."""
    if not spec.gathered_rows(len(rows)):
      if spec.mix == FusedSpec.BUCKETING:
        raise tools.UserException("Bucketing with s = %d reduces %d gradient rows to %d, not the rule's %d" % (
          spec.bucket_size, len(rows), -(-len(rows) // spec.bucket_size), spec.n))
      raise tools.UserException("Expected %d gradient rows, got %d" % (spec.n, len(rows)))
    if not 1 <= len(segments) <= MAX_SEGMENTS:
      raise tools.UserException("Between 1 and %d coordinate segments per rank (got %d)" % (MAX_SEGMENTS, len(segments)))
    addr = lambda t: 0 if t is None else (t if isinstance(t, int) else t.data_ptr())
    a = GarArgs(n=spec.n, f=spec.f, m=spec.m, beta=spec.beta, rule=spec.rule_id, n_rows=len(rows), bkt_size=spec.bucket_size or 0,
                bkt_seed=int(bucketing_seed), R=R, rank=rank, nseg=len(segments), first_seg=first_seg, seg_max_ctas=self.phase_a_ctas,
                grad_mc=int(grad_mc or 0), workers_per_rank=workers_per_rank, row_stride=row_stride, agg_out=addr(agg_out),
                opt=OPTIMIZERS[opt], lr=lr, h0=hyper[0], h1=hyper[1], h2=hyper[2], hyper_ptr=addr(hyper_ptr), param=addr(param),
                slot0=addr(slot0), slot1=addr(slot1), param_mc=int(param_mc or 0), epoch=epoch & 0x7fffffff, epoch_ptr=addr(epoch_ptr),
                cta_partials=self.cta_partials.data_ptr(), seg_partials=self.seg_partials.data_ptr(), staging=addr(staging),
                raw_dist_out=self.raw_dist_out.data_ptr(), info=self.info.data_ptr(), loss_in=addr(loss_in),
                nloss=loss_in.numel() if loss_in is not None else 0, loss_out=addr(loss_out), iterations=spec.iterations, nu=spec.nu,
                tau=spec.tau, center=addr(center), mix=spec.mix_id, arc_out=self.arc_out.data_ptr(), dnc_b=spec.subsample, dnc_step=step,
                dnc_seed=spec.seed, dnc_step_ptr=addr(step_ptr), root=addr(root), fltrust_out=self.fltrust_out.data_ptr(),
                history=addr(history), foolsgold_out=self.foolsgold_out.data_ptr(), confidence=spec.confidence)
    a.dist_out = (self.geo_dist_out if spec.rule in ITERATIVE_RULES else self.dnc_dist_out if spec.rule == "dnc" else self.dist_out).data_ptr()
    for s, (lo, hi) in enumerate(segments):
      a.seg_lo[s], a.seg_hi[s], a.seg_ctas[s] = lo, hi, self.phase_a_ctas if s < first_seg else 0
    for i, row in enumerate(rows):
      a.grad[i] = row
    for q in range(R):
      a.param_dst[q] = addr(param_dst[q]) if param_dst is not None else (addr(param) if q == 0 else 0)
      a.signal[q] = addr(signals[q]) if signals is not None else 0
      a.mailbox[q] = addr(mailboxes[q]) if mailboxes is not None else (self.local_mailbox.data_ptr() if q == 0 else 0)
      a.param_bf16_dst[q] = addr(param_bf16_dst[q]) if param_bf16_dst is not None else 0
    a.dnc_domain = max(hi for _, hi in segments) if domain is None else domain
    scratch = None
    if spec.rule == "dnc":
      a.dnc_r = spec.removed
      scratch = self.dnc_scratch(spec, a.dnc_domain)
      a.dnc_scratch = scratch.data_ptr()
    elif spec.rule == "smea":
      scratch = self.smea_scratch(spec)
      a.smea_scratch = scratch.data_ptr()
    return a, scratch.numel() if scratch is not None else 0

  def dnc_scratch(self, spec, domain):
    """DnC's scratch for rule `spec` over `domain` coordinates: the CTA partials of the sampled distances of the largest grid, then the
    gathered samples [T][n][b' rounded up to 4] (grown on demand)."""
    count = min(spec.subsample, int(domain))
    need = self.ctas * DNC_MAX_ITERATIONS * MAX_PAIRS + spec.iterations * spec.n * ((count + 3) // 4 * 4)
    if self._dnc_scratch is None or self._dnc_scratch.numel() < need:
      self._dnc_scratch = torch.zeros(need, dtype=torch.float32, device=self.device)
    return self._dnc_scratch

  def smea_scratch(self, spec):
    """SMEA's workspace for rule `spec`: one [m][m] float64 slab (m = n - f) per warp of the largest grid."""
    m = max(spec.n - spec.f, 0)
    need = self.ctas * ((512 if spec.n <= 8 else 256) // 32) * m * m
    if self._smea_scratch is None or self._smea_scratch.numel() < need:
      self._smea_scratch = torch.zeros(need, dtype=torch.float64, device=self.device)
    return self._smea_scratch

  def mimic_scratch(self, d):
    """Mimic's y scratch over d coordinates (grown on demand): y of a warm-up step, kept apart from z until its norm is known."""
    if self._mimic_y is None or self._mimic_y.numel() < d:
      self._mimic_y = torch.zeros(d, dtype=torch.float32, device=self.device)
    return self._mimic_y

  def launch(self, spec, rows, lo=None, hi=None, *, segments=None, stream=None, max_ctas_limit=0, **kwargs):
    """The finish kernel (the whole aggregation unless `first_seg` segments were pre-accumulated by `phase_a`).
    `rows`: n device addresses of the workers' gradient rows (raw ints, local or peer-mapped); owned coordinates `[lo, hi)` or `segments`."""
    args, scratch_elems = self._fill(spec, rows, segments if segments is not None else [(lo, hi)], **kwargs)
    with torch.cuda.device(self.device):
      _check(self._func(args, max_ctas_limit, scratch_elems, _stream_ptr(stream)), "gar_fused")

  def phase_a(self, spec, rows, segments, seg, *, stream=None, max_ctas_limit=0, **kwargs):
    """Pre-accumulate the partial distances of owned segment `seg` (and stage its tile) on a few CTAs, e.g. under the backward pass.
    Takes `launch`'s arguments; `max_ctas_limit` bounds the finish kernel alone."""
    args, _ = self._fill(spec, rows, segments, **kwargs)
    with torch.cuda.device(self.device):
      _check(self._phase_a(args, seg, self.phase_a_ctas, self.phase_a_threads, _stream_ptr(stream)), "gar_phase_a")


_launchers = {}


def _torch_rules(spec, step=0):
  from ..aggregators import _ops
  return {"average": _ops.torch_average, "average-nan": _ops.torch_average_nan, "median": _ops.torch_median,
          "averaged-median": lambda M: _ops.torch_averaged_median(M, spec.beta), "krum": lambda M: _ops.torch_krum(M, spec.f, spec.m),
          "bulyan": lambda M: _ops.torch_bulyan(M, spec.f, spec.m), "trimmed-mean": lambda M: _ops.torch_trimmed_mean(M, spec.f),
          "mda": lambda M: _ops.torch_mda(M, spec.f), "geometric-median": lambda M: _ops.torch_geometric_median(M, spec.iterations, spec.nu),
          "dnc": lambda M: _ops.torch_dnc(M, spec.f, spec.iterations, spec.subsample, spec.c, spec.seed, step),
          "smea": lambda M: _ops.torch_smea(M, spec.f)}[spec.rule]


def aggregate(spec, G, return_details=False, center=None, step=0, bucketing_seed=0, root=None, history=None):
  """Stand-alone aggregation of the CUDA matrix `G` ([n, d], fp32) with rule `spec` -> [d] tensor. `return_details` also returns the
  distances (Krum / Bulyan / MDA: the [n, n] matrix; geometric median, centered clipping: the [iterations, n] row distances of every
  iteration) and the selection masks. Centered clipping needs `center`, a [d] tensor of G's dtype on G's device, updated in place.
  DnC draws its samples with step key `step` over the d coordinates of G's rows; its details are the [T, n, n] sampled distances and
  `info` with [0] = 1, [1] = the final mask (bit i: row i kept) and [96 + t] = the mask of iteration t. SMEA's details are MDA's (the
  [n, n] distances and `info`), then its winning score (a 0-d float64 tensor).
  With `spec.mix == "nnm"` the rule runs on the mixed rows (its distances and masks are those of the mixed rows), and
  `return_details` adds a fourth element: (distances of the raw rows [n, n], NNM masks [n] int32). With "arc" the rule runs on the
  clipped rows and `return_details` adds (squared norms N [n], factors c [n]); with "arc+nnm" NNM mixes the clipped rows (its
  distances are theirs) and both elements follow, NNM's first.
  With "bucketing" G holds the n gathered rows and the rule runs on the n' = ceil(n / spec.bucket_size) bucket means, drawn with step
  key `step` and seed `bucketing_seed` (its distances and masks are those of the means); `return_details` adds (permutation [n] int32,
  bucket masks [n'] int32).
  FLTrust needs `root`, the [d] root gradient; its details are (P [n], N [n], N0, a [n]), CPU tensors: the kernel's sums and coefficients.
  FoolsGold needs `history`, the [n, d] per-worker histories of G's dtype on G's device, updated in place; its details are (P [n, n],
  N [n], bad [n] bool, c [n]), NumPy arrays: the kernel's sums of the updated histories, bad-row flags and coefficients."""
  if not G.is_cuda:
    raise tools.UserException("ops.gar.aggregate expects a CUDA tensor")
  from ..aggregators import _ops
  n, d = G.shape
  bucketing = spec.mix == FusedSpec.BUCKETING
  m = _ops.check_bucketing(n, spec.bucket_size) if bucketing else n   # the rows the rule sees
  if m != spec.n:
    spec = spec.with_rows(m)
  if spec.rule == "dnc":
    step = _ops.check_dnc_step(step)
  if bucketing:
    bucketing_seed, step = _ops.check_bucketing_key(bucketing_seed, step)
  if spec.rule == "centered-clipping":
    return _aggregate_centered_clipping(spec, G, return_details, center, step, bucketing_seed)
  if spec.rule == "fltrust":
    return _aggregate_fltrust(spec, G, return_details, root)
  if spec.rule == "foolsgold":
    return _aggregate_foolsgold(spec, G, return_details, history)
  if G.dtype == torch.float64 and not return_details:
    # the reference's ops are registered for double too (`native/op_krum/op.cpp:47`): the sm_90a kernels are fp32, so double inputs are
    # aggregated in double by the device-side torch implementations of the same rules (same ordering convention) instead of being rounded
    return _torch_rules(spec, step)(_torch_mixed(spec, G, step, bucketing_seed))
  if G.dtype != torch.float32:
    out = aggregate(spec, G.float(), return_details, step=step, bucketing_seed=bucketing_seed)
    return (out[0].to(G.dtype),) + out[1:] if return_details else out.to(G.dtype)
  if n > MAX_WORKERS:  # beyond the kernels' worker limit: torch ops on the same device
    return _torch_rules(spec, step)(_torch_mixed(spec, G, step, bucketing_seed))
  G, dp = _aligned_rows(G)
  launcher = _launcher(G.device, n, m)
  out = torch.empty(dp, dtype=torch.float32, device=G.device)
  rows = [G.data_ptr() + i * dp * 4 for i in range(n)]
  launcher.launch(spec, rows, 0, dp, agg_out=out, staging=_staging(spec, dp, G.device), step=step, domain=d, bucketing_seed=bucketing_seed)
  out = out[:d]
  if return_details:
    if spec.rule in ITERATIVE_RULES:
      dist = launcher.geo_dist_out[:spec.iterations * m].view(spec.iterations, m)
    elif spec.rule == "dnc":
      dist = launcher.dnc_dist_out[:spec.iterations * m * m].view(spec.iterations, m, m)
    else:
      dist = launcher.dist_out[:m * m].view(m, m)
    info = launcher.info.clone()
    score = (info[32:34].cpu().view(torch.float64)[0],) if spec.rule == "smea" else ()
    return (out, dist.clone(), info) + score + _mix_details(spec, launcher, n)
  return out


def _padded(t, dp):
  """The [d] vector or [n, d] matrix `t` itself when d = dp and it is contiguous on a 16-byte boundary, else a zero-padded [.., dp] copy.
  A caller whose kernel writes the buffer copies [.., :d] back into `t` when it received a copy."""
  d = t.shape[-1]
  if d == dp and t.is_contiguous() and t.data_ptr() % 16 == 0:
    return t
  copy = torch.zeros(t.shape[:-1] + (dp,), dtype=t.dtype, device=t.device)
  copy[..., :d] = t
  return copy


def _aligned_rows(G):
  """`_padded` rows of the [n, d] matrix G, dp the next multiple of 4 -> (rows, dp)."""
  dp = G.shape[1] + (-G.shape[1]) % 4
  return _padded(G, dp), dp


def _staging(spec, dp, device):
  """NNM mixes and ARC clips the rows in place in a local [n, dp] tile, bucketing stores its n' means there: the stand-alone op has to
  provide one (of the rule's spec.n rows)."""
  return torch.empty((spec.n, dp), dtype=torch.float32, device=device) if spec.mix is not None else None


def _mix_details(spec, launcher, n):
  """The `return_details` elements of the pre-aggregation over n gathered rows: with NNM (raw distances [n, n], NNM masks [n] int32),
  then with ARC (squared norms [n], factors [n]); with bucketing (permutation [n] int32, bucket masks [n'] int32)."""
  if spec.mix == FusedSpec.BUCKETING:
    return ((launcher.info[128:128 + n].clone(), launcher.info[160:160 + spec.n].clone()),)
  details = ()
  if spec.mix_id & FusedSpec.MIX_NNM:
    details += ((launcher.raw_dist_out.view(n, n).clone(), launcher.info[64:64 + n].clone()),)
  if spec.mix_id & FusedSpec.MIX_ARC:
    arc = launcher.arc_out.clone()
    details += ((arc[:n], arc[n:]),)
  return details


def _torch_mixed(spec, G, step=0, bucketing_seed=0):
  """The fall-backs' pre-aggregation: `spec.mix` with the torch reference on G's device."""
  from ..aggregators import _ops
  return _ops.torch_pre_aggregate(G, spec.mix, spec.f, bucket_size=spec.bucket_size, seed=bucketing_seed, step=step)


def _launcher(device, n, rule_rows=None):
  """The cached launcher for n gathered rows; with bucketing one per rule row count too, since the kernels leave the diagonal of the
  [n', n'] distance view untouched (+0 from the allocation) and a view of another size would see other entries there."""
  key = (device.index, n) if rule_rows in (None, n) else (device.index, n, rule_rows)
  launcher = _launchers.get(key)
  if launcher is None:
    launcher = _launchers[key] = FusedLauncher(device, n)
  return launcher


def _aggregate_centered_clipping(spec, G, return_details, center, step=0, bucketing_seed=0):
  """`aggregate` for centered clipping: the sm_90a kernel for fp32 and n <= 32, the torch reference on the device otherwise."""
  from ..aggregators import _ops
  n, d = G.shape
  m = spec.n   # the rows the rule sees
  if center is None or center.shape != (d,) or center.device != G.device:
    raise tools.UserException("Centered clipping needs a [%d] center on %s" % (d, G.device))
  if G.dtype == torch.float64 or n > MAX_WORKERS:
    if center.dtype != G.dtype:
      raise tools.UserException("Centered clipping needs a center of type %s (got %s)" % (G.dtype, center.dtype))
    if return_details:
      raise tools.UserException("Centered clipping returns its details from the sm_90a kernel only (fp32, n <= %d)" % MAX_WORKERS)
    return _ops.torch_centered_clipping(_torch_mixed(spec, G, step, bucketing_seed), spec.iterations, spec.tau, center)
  if G.dtype != torch.float32 or center.dtype != torch.float32:
    raise tools.UserException("Centered clipping on the device needs fp32 rows and center (got %s, %s)" % (G.dtype, center.dtype))
  G, dp = _aligned_rows(G)
  work = _padded(center, dp)
  launcher = _launcher(G.device, n, m)
  out = torch.empty(dp, dtype=torch.float32, device=G.device)
  rows = [G.data_ptr() + i * dp * 4 for i in range(n)]
  launcher.launch(spec, rows, 0, dp, agg_out=out, center=work, staging=_staging(spec, dp, G.device), step=step, bucketing_seed=bucketing_seed)
  if work is not center:
    center.copy_(work[:d])
  out = out[:d]
  if return_details:
    dist = launcher.geo_dist_out[:spec.iterations * m].view(spec.iterations, m)
    return (out, dist.clone(), launcher.info.clone()) + _mix_details(spec, launcher, n)
  return out


def _aggregate_fltrust(spec, G, return_details, root):
  """`aggregate` for FLTrust: the sm_90a kernel for fp32 and n <= 32, the torch reference on the device otherwise (double rows in
  double)."""
  from ..aggregators import _ops
  n, d = G.shape
  if spec.mix is not None:
    raise tools.UserException("FLTrust takes no pre-aggregation (got %r)" % (spec.mix,))
  root = _ops.check_fltrust_root(G, root)
  if G.dtype == torch.float64 or n > MAX_WORKERS:
    if return_details:
      raise tools.UserException("FLTrust returns its details from the sm_90a kernel only (fp32, n <= %d)" % MAX_WORKERS)
    return _ops.torch_fltrust(G, root)
  if G.dtype != torch.float32:
    out = _aggregate_fltrust(spec, G.float(), return_details, root.float())
    return (out[0].to(G.dtype),) + out[1:] if return_details else out.to(G.dtype)
  G, dp = _aligned_rows(G)
  launcher = _launcher(G.device, n)
  out = torch.empty(dp, dtype=torch.float32, device=G.device)
  rows = [G.data_ptr() + i * dp * 4 for i in range(n)]
  staging = torch.empty((n, dp), dtype=torch.float32, device=G.device) if n > 8 else None   # beyond one 8-row block: the staged rows
  launcher.launch(spec, rows, 0, dp, agg_out=out, staging=staging, root=_padded(root, dp))
  out = out[:d]
  if return_details:
    fo = launcher.fltrust_out.cpu()
    return out, fo[:n].clone(), fo[MAX_WORKERS:MAX_WORKERS + n].clone(), fo[2 * MAX_WORKERS].clone(), fo[2 * MAX_WORKERS + 1:2 * MAX_WORKERS + 1 + n].clone()
  return out


def _aggregate_foolsgold(spec, G, return_details, history):
  """`aggregate` for FoolsGold: the sm_90a kernel for fp32 and n <= 32, the torch reference on the device otherwise (double rows in
  double)."""
  from ..aggregators import _ops
  n, d = G.shape
  if spec.mix is not None:
    raise tools.UserException("FoolsGold takes no pre-aggregation (got %r)" % (spec.mix,))
  history = _ops.check_foolsgold_history(G, history)
  if G.dtype == torch.float64 or n > MAX_WORKERS:
    if return_details:
      raise tools.UserException("FoolsGold returns its details from the sm_90a kernel only (fp32, n <= %d)" % MAX_WORKERS)
    return _ops.torch_foolsgold(G, history, spec.confidence)
  if G.dtype != torch.float32:
    raise tools.UserException("FoolsGold on the device needs fp32 or float64 rows (got %s)" % (G.dtype,))
  G, dp = _aligned_rows(G)
  work = _padded(history, dp)
  launcher = _launcher(G.device, n)
  out = torch.empty(dp, dtype=torch.float32, device=G.device)
  rows = [G.data_ptr() + i * dp * 4 for i in range(n)]
  staging = torch.empty((n, dp), dtype=torch.float32, device=G.device) if n > 8 else None   # beyond one 8-row block: the staged rows
  launcher.launch(spec, rows, 0, dp, agg_out=out, staging=staging, history=work)
  if work is not history:
    history.copy_(work[:, :d])
  out = out[:d]
  if return_details:
    return (out,) + foolsgold_details(launcher, n)
  return out


def foolsgold_details(launcher, n):
  """FoolsGold's (P [n, n], N [n], bad [n] bool, c [n] float32) of the launcher's last launch, as NumPy arrays (a synchronisation)."""
  import numpy as np
  fo = launcher.foolsgold_out.cpu().numpy()
  P = np.zeros((n, n), dtype=np.float32)
  iu = np.triu_indices(n)
  P[iu] = fo[:n * (n + 1) // 2]
  P.T[iu] = fo[:n * (n + 1) // 2]
  return P, np.diagonal(P).copy(), fo[FOOLSGOLD_SUMS:FOOLSGOLD_SUMS + n] != 0, fo[FOOLSGOLD_SUMS + MAX_WORKERS:FOOLSGOLD_SUMS + MAX_WORKERS + n].copy()


def worker_momentum_(G, M, beta, c):
  """Worker momentum on the [w, d] rows `G` and momenta `M`, in place: M <- beta * M + c * G, then G <- M, one rounding per operation.
  CUDA fp32 tensors run the sm_90a kernel (one launch for the w rows; G's rows may be strided); others the torch reference."""
  from ..aggregators import _ops
  if G.dim() != 2 or G.shape != M.shape:
    raise tools.UserException("Worker momentum needs [w, d] rows and momenta of the same shape (got %s, %s)" % (tuple(G.shape), tuple(M.shape)))
  if not G.is_cuda or G.dtype != torch.float32:
    return _ops.torch_worker_momentum_(G, M, beta, c)
  if M.dtype != torch.float32 or M.device != G.device:
    raise tools.UserException("Worker momentum needs fp32 momenta on the rows' device (got %s on %s)" % (M.dtype, M.device))
  w, d = G.shape
  if d > 1 and (G.stride(1) != 1 or M.stride(1) != 1):
    raise tools.UserException("Worker momentum needs rows with contiguous elements")
  func = _lib().agb_worker_momentum
  with torch.cuda.device(G.device):
    _check(func(ctypes.c_void_p(G.data_ptr()), ctypes.c_longlong(G.stride(0) if w > 1 else d), ctypes.c_void_p(M.data_ptr()),
                ctypes.c_longlong(M.stride(0) if w > 1 else d), ctypes.c_longlong(w), ctypes.c_longlong(d), ctypes.c_float(beta), ctypes.c_float(c),
                _stream_ptr()), "worker_momentum")
  return G


def craft(rows, segments, honest, byzantine, mode, coef, *, deviation=None, launcher=None, mailboxes=None, R=1, rank=0, signals=None, epoch=1,
          epoch_ptr=None, stream=None, state=None, warmup=None, f=None, threshold=None, scale=None, seed=None, step=None, search=True):
  """Craft the omniscient Byzantine rows (`attacks/omniscient.py`) over the owned `segments` of the n rows at device addresses `rows`
  (raw ints, local or peer-mapped): every slot of `byzantine` receives the ALIE / IPM / Min-Max / Min-Sum value of the `honest` slots.
  Collective when R > 1 (entry barrier through the signal pads, at flag value `epoch`, or `*epoch_ptr + 1` when given).
  Min-Max and Min-Sum (`coef` unused) take the `deviation` (default "unit-vec") and the `FusedLauncher` whose scratch holds the CTA
  partials and receives gamma and the summed statistics (`launcher.craft_stats`); their statistics are exchanged through `mailboxes`
  (R addresses, every rank's; default: the launcher's local mailbox when R = 1).
  Mimic (`coef` unused) takes the caller-owned `state` (`aggregators._ops.mimic_state`: "t", the fp32 "z" of the owned coordinates,
  `segments` back to back, and the [1] int32 "istar", both on the device) and the warm-up length `warmup`: while state["t"] < warmup it runs one
  warm-up update (two exchanges through `mailboxes`, the launcher's scratch; `launcher.mimic_stats` receives s_i, q_i, ||y||^2 and
  1 / ||y||) and counts it in state["t"]; then the copy pass alone, with i* read on the device.
  fang-krum (`coef` unused) takes the rule's declared `f` and the `threshold` (default `_ops.FANG_THRESHOLD`), and the launcher and
  mailboxes as Min-Max; `launcher.craft_stats` receives gamma and the summed statistics, `launcher.fang_out` gamma_max, t and the
  selected flag. `search=False` skips the candidate search (gamma = gamma_max): the passes alone, for timing. fang-trim (`coef` unused)
  takes the `scale` beta (default `_ops.FANG_SCALE`), the `seed` and the `step` key; it exchanges nothing."""
  from ..aggregators import _ops
  n = len(rows)
  if n > MAX_WORKERS:
    raise tools.UserException("The sm_90a crafting kernel supports n <= %d workers (got %d)" % (MAX_WORKERS, n))
  if not 1 <= len(segments) <= MAX_SEGMENTS:
    raise tools.UserException("Between 1 and %d coordinate segments per rank (got %d)" % (MAX_SEGMENTS, len(segments)))
  mask = lambda slots: sum(1 << int(i) for i in set(slots))
  addr = lambda t: 0 if t is None else (t if isinstance(t, int) else t.data_ptr())
  c_rows = (ctypes.c_ulonglong * n)(*[int(r) for r in rows])
  lo = (ctypes.c_longlong * len(segments))(*[int(a) for a, _ in segments])
  hi = (ctypes.c_longlong * len(segments))(*[int(b) for _, b in segments])
  c_signals = (ctypes.c_ulonglong * R)(*[addr(signals[q]) for q in range(R)]) if signals is not None else None
  # the leading and trailing arguments of every crafting entry point
  rows_args = (c_rows, ctypes.c_int(n), lo, hi, ctypes.c_int(len(segments)), ctypes.c_uint(mask(honest)), ctypes.c_uint(mask(byzantine)))
  epoch_args = (ctypes.c_uint(epoch & 0x7fffffff), ctypes.c_ulonglong(addr(epoch_ptr)), _stream_ptr(stream))
  if mode == "fang-krum":
    threshold = _ops.check_fang_krum(n, len(set(byzantine)), f, threshold)
  elif mode in ("min-max", "min-sum"):
    if deviation is None:
      deviation = "unit-vec"
    if deviation not in DEVIATIONS:
      raise tools.UserException("Unknown deviation %r for %s (expected one of %s)" % (deviation, mode, ", ".join(DEVIATIONS)))
  if mode in ("mimic", "fang-krum", "min-max", "min-sum"):   # the launcher's scratch, and a cross-rank exchange through the mailboxes
    if launcher is None or (mode == "mimic" and (state is None or warmup is None)):
      raise tools.UserException(mode + " needs the scratch of a FusedLauncher" + (", its state and its warm-up length" if mode == "mimic" else ""))
    if mailboxes is None:
      if R != 1:
        raise tools.UserException("%s over %d ranks needs every rank's mailbox" % (mode, R))
      mailboxes = [launcher.local_mailbox]
    c_mailboxes = (ctypes.c_ulonglong * R)(*[addr(mailboxes[q]) for q in range(R)])
  if mode == "mimic":
    t = int(state["t"])
    warm = t < int(warmup)
    z = state["z"]
    if z.numel() != sum(int(b) - int(a) for a, b in segments):
      raise tools.UserException("mimic's z holds the %d owned coordinates (got %d)" % (sum(int(b) - int(a) for a, b in segments), z.numel()))
    y = launcher.mimic_scratch(z.numel()) if warm else None
    func = _lib().agb_gar_byzantine_mimic
    func.restype = ctypes.c_int
    _check(func(*rows_args, ctypes.c_int(1 if warm else 0), ctypes.c_int(t), ctypes.c_int(R), ctypes.c_int(rank), c_signals, c_mailboxes,
                ctypes.c_ulonglong(launcher.craft_partials.data_ptr()), ctypes.c_int(launcher.craft_ctas), ctypes.c_ulonglong(addr(z)),
                ctypes.c_ulonglong(addr(y)), ctypes.c_ulonglong(addr(state["istar"])), ctypes.c_ulonglong(launcher.mimic_stats.data_ptr()),
                *epoch_args), "gar_byzantine_mimic")
    if warm:
      state["t"] = t + 1
    return
  if mode == "fang-trim":
    scale = _ops.check_fang_scale(scale)
    key = _ops.fang_trim_key(0 if seed is None else seed, step)
    func = _lib().agb_gar_byzantine_fang_trim
    func.restype = ctypes.c_int
    _check(func(*rows_args, ctypes.c_float(scale), ctypes.c_ulonglong(key), ctypes.c_int(R), ctypes.c_int(rank), c_signals, *epoch_args),
           "gar_byzantine_fang_trim")
    return
  if mode == "fang-krum":
    func = _lib().agb_gar_byzantine_fang_krum
    func.restype = ctypes.c_int
    _check(func(*rows_args, ctypes.c_int(f), ctypes.c_float(threshold), ctypes.c_int(1 if search else 0), ctypes.c_int(R), ctypes.c_int(rank),
                c_signals, c_mailboxes,
                ctypes.c_ulonglong(launcher.craft_partials.data_ptr()), ctypes.c_int(launcher.craft_ctas), ctypes.c_ulonglong(launcher.craft_stats.data_ptr()),
                ctypes.c_ulonglong(launcher.fang_out.data_ptr()), *epoch_args), "gar_byzantine_fang_krum")
    return
  if mode in ("min-max", "min-sum"):
    func = _lib().agb_gar_byzantine_optimized
    func.restype = ctypes.c_int
    _check(func(*rows_args, ctypes.c_int(BYZANTINE_MODES[mode]), ctypes.c_int(DEVIATIONS[deviation]), ctypes.c_int(R), ctypes.c_int(rank),
                c_signals, c_mailboxes,
                ctypes.c_ulonglong(launcher.craft_partials.data_ptr()), ctypes.c_int(launcher.craft_ctas), ctypes.c_ulonglong(launcher.craft_stats.data_ptr()),
                *epoch_args), "gar_byzantine_optimized")
    return
  func = _lib().agb_gar_byzantine
  func.restype = ctypes.c_int
  _check(func(*rows_args, ctypes.c_int(BYZANTINE_MODES[mode]), ctypes.c_float(coef), ctypes.c_int(R), ctypes.c_int(rank), c_signals,
              *epoch_args), "gar_byzantine")


def craft_details(launcher, mode, H):
  """(gamma, A [H], B [H], C, T) of the last Min-Max / Min-Sum crafting run with `launcher`: Python floats (fp32 values), as the kernel
  solved them; T is None for Min-Sum."""
  stats = launcher.craft_stats.cpu().tolist()
  st = stats[1:]
  a, b, c = MAX_PAIRS, MAX_PAIRS + MAX_WORKERS, MAX_PAIRS + 2 * MAX_WORKERS
  T = max(st[:H * (H - 1) // 2]) if mode == "min-max" else None
  return stats[0], st[a:a + H], st[b:b + H], st[c], T


def fang_krum_details(launcher, H):
  """(gamma, selected, t, gamma_max, A [H], B [H], C, T [H (H - 1) / 2]) of the last fang-krum crafting run with `launcher`, as the kernel
  solved them: the sums are fp32 values, gamma_max a float64 value, T the honest pair distances in pair order."""
  stats = launcher.craft_stats.cpu().tolist()
  gamma_max, t, selected = launcher.fang_out.cpu().tolist()
  st = stats[1:]
  a, b, c = MAX_PAIRS, MAX_PAIRS + MAX_WORKERS, MAX_PAIRS + 2 * MAX_WORKERS
  return stats[0], bool(selected), int(t), gamma_max, st[a:a + H], st[b:b + H], st[c], st[:H * (H - 1) // 2]


def mimic_details(launcher, H):
  """(s [H], q [H], ||y||^2, 1 / ||y||) of the last mimic warm-up step run with `launcher`: Python floats, as the kernel summed them (s and
  1 / ||y|| are fp32 values)."""
  stats = launcher.mimic_stats.cpu().tolist()
  return stats[:H], stats[MAX_WORKERS:MAX_WORKERS + H], stats[2 * MAX_WORKERS], stats[2 * MAX_WORKERS + 1]


def _craft_mimic_(G, byz_slots, state, warmup, return_details):
  """`craft_byzantine_` for mimic: the sm_90a kernels on CUDA fp32 rows with n <= 32, the torch reference otherwise."""
  from ..aggregators import _ops
  n, d = G.shape
  slots, warmup = _ops.check_mimic(n, byz_slots, warmup)
  if state is None or state["z"].shape != (d,) or state["z"].dtype != torch.float32 or state["z"].device != G.device or state["istar"].device != G.device:
    raise tools.UserException("mimic needs a state with an fp32 [%d] z and its target on %s (`aggregators._ops.mimic_state`)" % (d, G.device))
  if not G.is_cuda or n > MAX_WORKERS:
    return _ops.torch_mimic_step_(G, slots, state, warmup, return_details=return_details)
  if G.dtype != torch.float32:
    raise tools.UserException("ops.gar.craft_byzantine_ expects fp32 rows (got %s)" % G.dtype)
  work, dp = _aligned_rows(G)
  z = state["z"]
  zwork = _padded(z, dp)
  run = dict(state, z=zwork)
  warm = run["t"] < warmup
  launcher = _launcher(G.device, n)
  rows = [work.data_ptr() + i * dp * 4 for i in range(n)]
  with torch.cuda.device(G.device):
    craft(rows, [(0, dp)], [i for i in range(n) if i not in slots], slots, "mimic", None, launcher=launcher, state=run, warmup=warmup)
  state["t"] = run["t"]
  if zwork is not z:
    z.copy_(zwork[:d])
  if work is not G:
    index = torch.tensor(slots, dtype=torch.int64, device=G.device)
    G[index] = work[index, :d]
  if return_details:
    return mimic_details(launcher, n - len(slots)) if warm else None
  return G


def craft_byzantine_(G, byz_slots, mode, coef=None, deviation=None, return_details=False, state=None, warmup=None, f=None, threshold=None,
                     scale=None, seed=None, step=None):
  """Stand-alone omniscient attack on the [n, d] fp32 matrix `G`, in place: rows `byz_slots` <- the ALIE (`coef` = z), IPM
  (`coef` = epsilon), Min-Max or Min-Sum (`deviation`) row of the other rows. CUDA tensors with n <= 32 run the sm_90a kernel; others
  the torch reference. Min-Max / Min-Sum with `return_details` return (gamma, A, B, C, T) instead of G (see `craft_details`).
  Mimic takes its `state` (`aggregators._ops.mimic_state(d, G.device)`, updated in place) and `warmup`; with `return_details` it returns
  (s, q, ||y||^2, 1 / ||y||) of a warm-up step (see `mimic_details`), None after the warm-up.
  fang-krum needs the rule's declared `f` and takes `threshold`; with `return_details` it returns (gamma, selected, t, gamma_max, A, B, C,
  T) (see `fang_krum_details`). fang-trim takes `scale`, `seed` (default 0) and the `step` key (required); the column index of G is the
  coordinate x of its draw."""
  from ..aggregators import _ops
  if mode == "mimic":
    return _craft_mimic_(G, byz_slots, state, warmup, return_details)
  n, d = G.shape
  byz_slots = _ops.check_byzantine_slots(n, byz_slots, mode)
  optimized = mode in _ops.OPTIMIZED_MODES
  fang = dict(f=f, threshold=threshold, scale=scale, seed=0 if seed is None else seed, step=step)
  if optimized:
    deviation = _ops.check_deviation(mode, deviation)
  elif mode == "fang-krum":
    _ops.check_fang_krum(n, len(byz_slots), f, threshold)
  elif mode == "fang-trim":
    _ops.check_fang_scale(scale)
    _ops.fang_trim_key(fang["seed"], step)
    if return_details:
      raise tools.UserException("return_details is for Min-Max / Min-Sum / fang-krum only")
  elif return_details:
    raise tools.UserException("return_details is for Min-Max / Min-Sum / fang-krum only")
  if not G.is_cuda or n > MAX_WORKERS:
    return _ops.torch_craft_byzantine_(G, byz_slots, mode, coef, deviation=deviation, return_details=return_details, **fang)
  if G.dtype != torch.float32:
    raise tools.UserException("ops.gar.craft_byzantine_ expects fp32 rows (got %s)" % G.dtype)
  work, dp = _aligned_rows(G)
  rows = [work.data_ptr() + i * dp * 4 for i in range(n)]
  launcher = _launcher(G.device, n) if optimized or mode == "fang-krum" else None
  with torch.cuda.device(G.device):
    craft(rows, [(0, dp)], [i for i in range(n) if i not in byz_slots], byz_slots, mode, coef, deviation=deviation, launcher=launcher, **fang)
  if work is not G:
    index = torch.tensor(byz_slots, dtype=torch.int64, device=G.device)
    G[index] = work[index, :d]
  if return_details:
    if mode == "fang-krum":
      return fang_krum_details(launcher, n - len(byz_slots))
    return craft_details(launcher, mode, n - len(byz_slots))
  return G


def sgd_(param, grad, lr):
  """In-place `param -= lr * grad` on flat fp32 CUDA buffers (baseline path's separate update kernel)."""
  func = _lib().agb_sgd
  _check(func(ctypes.c_void_p(param.data_ptr()), ctypes.c_void_p(grad.data_ptr()), ctypes.c_float(lr), ctypes.c_longlong(param.numel()), _stream_ptr()), "sgd")
  return param


def drop_chunks_(grad, rate, mode="nan", previous=None, chunk_bytes=65000, seed=0):
  """Lossy-transport emulation on a flat fp32 CUDA gradient: lost 65 000-byte chunks -> NaN / zero / previous bytes."""
  modes = {"nan": 0, "zero": 1, "clever": 2}
  func = _lib().agb_drop_chunks
  _check(func(ctypes.c_void_p(grad.data_ptr()), ctypes.c_void_p(previous.data_ptr() if previous is not None else 0), ctypes.c_longlong(grad.numel()),
              ctypes.c_longlong(chunk_bytes), ctypes.c_float(rate), ctypes.c_int(modes[mode]), ctypes.c_ulonglong(seed & (2 ** 64 - 1)), _stream_ptr()), "drop_chunks")
  return grad


def checksum(tensor):
  """64-bit position-dependent checksum of a flat fp32 CUDA buffer (cross-rank equality debug mode)."""
  out = torch.zeros(1, dtype=torch.int64, device=tensor.device)
  func = _lib().agb_checksum
  _check(func(ctypes.c_void_p(tensor.data_ptr()), ctypes.c_longlong(tensor.numel()), ctypes.c_void_p(out.data_ptr()), _stream_ptr()), "checksum")
  return out


def sha256_tree_host(data):
  """The digest `sha256` computes, on host bytes: a SHA-256 tree over 1024-byte leaves, every node hashed with a (level, index) header
  (`native/op_gar/digest.cu`)."""
  import hashlib
  import struct
  level, buf = 0, bytes(data)
  while True:
    count = max(1, (len(buf) + 1023) // 1024)
    nodes = [hashlib.sha256(struct.pack("<IIQ", level, 0, i) + buf[i * 1024:(i + 1) * 1024]).digest() for i in range(count)]
    if count == 1:
      return nodes[0]
    level, buf = level + 1, b"".join(nodes)


_sha_scratch = {}


def sha256(tensor):
  """SHA-256 tree digest (32 bytes, uint8 tensor on the same device) of a contiguous CUDA tensor whose size is a multiple of 4 bytes:
  the cryptographic digest signed by gradient authentication."""
  if not tensor.is_contiguous():
    tensor = tensor.contiguous()
  nbytes = tensor.numel() * tensor.element_size()
  lib = _lib()
  lib.agb_sha256_scratch_bytes.restype = ctypes.c_longlong
  need = int(lib.agb_sha256_scratch_bytes(ctypes.c_longlong(nbytes)))
  scratch = _sha_scratch.get(tensor.device)
  if scratch is None or scratch.numel() < need:
    scratch = _sha_scratch[tensor.device] = torch.empty(max(need, 1 << 20), dtype=torch.uint8, device=tensor.device)
  out = torch.empty(32, dtype=torch.uint8, device=tensor.device)
  _check(lib.agb_sha256_tree(ctypes.c_void_p(tensor.data_ptr()), ctypes.c_longlong(nbytes), ctypes.c_void_p(scratch.data_ptr()), ctypes.c_void_p(out.data_ptr()), _stream_ptr()), "sha256_tree")
  return out


def cast_bf16_(src, dst):
  """fp32 -> bf16 copy of a flat buffer (compute copy of the master parameters)."""
  func = _lib().agb_cast_bf16
  _check(func(ctypes.c_void_p(src.data_ptr()), ctypes.c_void_p(dst.data_ptr()), ctypes.c_longlong(src.numel()), _stream_ptr()), "cast_bf16")
  return dst

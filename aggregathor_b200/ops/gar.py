"""Python front-end of the sm_90a aggregation kernels (`native/op_gar`).

`aggregate(spec, G)` is the stand-alone `[n, d] -> [d]` custom op (the `-co` flavour of
the reference, which only ever had a CPU kernel: `native/op_krum/op.cpp:98-107`).
`FusedLauncher` drives the full gather + rule + optimizer + broadcast kernel for one rank
(see `parallel/fused.py` for the multi-GPU wiring).
"""

import ctypes
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
FLAG_SLOTS = MAX_SEGMENTS + 3 + MAX_ITERATIONS   # per segment: bucket entry; then exchange, exit, Byzantine crafting entry; one per iteration
SIGNAL_BYTES = FLAG_SLOTS * MAX_RANKS * 4
MAILBOX_BYTES = MAX_RANKS * (MAX_PAIRS + 1) * 4
OPTIMIZERS = {"none": 0, "sgd": 1, "adam": 2, "rmsprop": 3, "adagrad": 4, "adadelta": 5}

_ERRORS = {
  100: "unsupported number of workers/ranks (n <= 32, R <= 16)", 101: "segment bounds must be multiples of 4 elements (at most 8 segments)",
  102: "unknown rule", 103: "invalid Krum parameters", 104: "invalid Bulyan parameters", 105: "invalid beta",
  106: "optimizer requested without parameter buffers", 107: "optimizer slots missing", 108: "scratch buffers missing",
  109: "signal pads missing", 110: "more than 8 workers over several ranks need the staging buffer", 111: "invalid phase A launch",
  112: "invalid trimmed-mean parameters (0 <= 2 f < n)", 113: "invalid MDA parameters (0 <= 2 f < n and C(n, f) <= 2^20)",
  114: "invalid Byzantine crafting parameters (disjoint slot masks, at least one Byzantine slot, H >= 2 for ALIE, H >= 1 for IPM)",
  115: "invalid geometric-median parameters (0 <= 2 f < n, 1 <= iterations <= 16, finite nu > 0)",
  116: "invalid centered-clipping parameters (0 <= 2 f < n, 1 <= iterations <= 16, finite tau > 0, a center buffer)"}
ITERATIVE_RULES = ("geometric-median", "centered-clipping")   # [iterations, n] row distances in `geo_dist_out`
BYZANTINE_MODES = {"alie": 0, "ipm": 1}


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


class FusedLauncher:
  """Holds the scratch buffers and argument arrays of one rank's fused aggregation kernels (phase A kernels + finish kernel)."""

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
    self.local_mailbox = torch.zeros(MAILBOX_BYTES // 4, dtype=torch.float32, device=self.device)
    self.dist_out = torch.zeros(n * n, dtype=torch.float32, device=self.device)
    self.geo_dist_out = torch.zeros(MAX_ITERATIONS * n, dtype=torch.float32, device=self.device)   # iterative rules: D of every iteration, [T, n]
    self.info = torch.zeros(64, dtype=torch.int32, device=self.device)
    self._ptrs = (ctypes.c_ulonglong * 112)()
    self._ints = (ctypes.c_int * 32)()
    self._longs = (ctypes.c_longlong * (1 + 2 * MAX_SEGMENTS))()
    self._floats = (ctypes.c_float * 6)()
    self._func = _lib().agb_gar_fused
    self._func.restype = ctypes.c_int
    self._phase_a = _lib().agb_gar_phase_a
    self._phase_a.restype = ctypes.c_int
    timeout = os.environ.get("AGB_FLAG_TIMEOUT_S")
    if timeout is not None:   # bound of the cross-GPU flag waits (default 120 s, 0 = wait forever)
      with torch.cuda.device(self.device):
        _check(_lib().agb_gar_set_flag_timeout(ctypes.c_double(float(timeout))), "gar_set_flag_timeout")

  def _fill(self, spec, rows, segments, *, agg_out=None, opt="none", lr=0.0, hyper=(0.0, 0.0, 0.0), param=None, slot0=None, slot1=None, param_dst=None, param_mc=0,
            param_bf16_dst=None, rank=0, R=1, signals=None, mailboxes=None, epoch=1, staging=None, max_ctas_limit=0, grad_mc=0, workers_per_rank=1, row_stride=0,
            first_seg=0, epoch_ptr=None, hyper_ptr=None, loss_in=None, loss_out=None, center=None):
    ptrs = self._ptrs
    for i in range(112):
      ptrs[i] = 0
    if len(rows) != spec.n:
      raise tools.UserException("Expected %d gradient rows, got %d" % (spec.n, len(rows)))
    if not 1 <= len(segments) <= MAX_SEGMENTS:
      raise tools.UserException("Between 1 and %d coordinate segments per rank (got %d)" % (MAX_SEGMENTS, len(segments)))
    for i, row in enumerate(rows):
      ptrs[i] = row
    addr = lambda t: 0 if t is None else (t if isinstance(t, int) else t.data_ptr())
    ptrs[32], ptrs[33], ptrs[34], ptrs[35], ptrs[36] = addr(agg_out), addr(param), addr(slot0), addr(slot1), int(param_mc or 0)
    dist_out = self.geo_dist_out if spec.rule in ITERATIVE_RULES else self.dist_out
    ptrs[37], ptrs[38], ptrs[39], ptrs[40], ptrs[41] = self.cta_partials.data_ptr(), addr(staging), dist_out.data_ptr(), self.info.data_ptr(), int(grad_mc or 0)
    ptrs[42], ptrs[43], ptrs[44], ptrs[45], ptrs[46] = addr(epoch_ptr), addr(hyper_ptr), self.seg_partials.data_ptr(), addr(loss_in), addr(loss_out)
    ptrs[47] = addr(center)
    for q in range(R):
      ptrs[48 + q] = addr(param_dst[q]) if param_dst is not None else (addr(param) if q == 0 else 0)
      ptrs[64 + q] = addr(signals[q]) if signals is not None else 0
      ptrs[80 + q] = addr(mailboxes[q]) if mailboxes is not None else (self.local_mailbox.data_ptr() if q == 0 else 0)
      ptrs[96 + q] = addr(param_bf16_dst[q]) if param_bf16_dst is not None else 0
    ints = self._ints
    ints[0], ints[1], ints[2], ints[3], ints[4] = spec.n, spec.f, spec.m, spec.beta, spec.rule_id
    ints[5], ints[6], ints[7], ints[8], ints[9] = R, rank, OPTIMIZERS[opt], epoch & 0x7fffffff, max_ctas_limit
    ints[10], ints[11], ints[12], ints[13] = workers_per_rank, len(segments), first_seg, (loss_in.numel() if loss_in is not None else 0)
    ints[14], ints[15], ints[24], ints[25] = self.phase_a_ctas, self.phase_a_ctas, self.phase_a_threads, spec.iterations
    self._longs[0] = row_stride
    for s in range(MAX_SEGMENTS):
      lo, hi = segments[s] if s < len(segments) else (0, 0)
      self._longs[1 + s], self._longs[1 + MAX_SEGMENTS + s] = lo, hi
      ints[16 + s] = self.phase_a_ctas if s < first_seg else 0
    self._floats[0], self._floats[1], self._floats[2], self._floats[3], self._floats[4] = lr, hyper[0], hyper[1], hyper[2], spec.nu
    self._floats[5] = spec.tau

  def launch(self, spec, rows, lo=None, hi=None, *, segments=None, stream=None, **kwargs):
    """The finish kernel (the whole aggregation unless `first_seg` segments were pre-accumulated by `phase_a`).
    `rows`: n device addresses of the workers' gradient rows (raw ints, local or peer-mapped); owned coordinates `[lo, hi)` or `segments`."""
    self._fill(spec, rows, segments if segments is not None else [(lo, hi)], **kwargs)
    with torch.cuda.device(self.device):
      _check(self._func(self._ptrs, self._ints, self._longs, self._floats, _stream_ptr(stream)), "gar_fused")

  def phase_a(self, spec, rows, segments, seg, *, stream=None, **kwargs):
    """Pre-accumulate the partial distances of owned segment `seg` (and stage its tile) on a few CTAs, e.g. under the backward pass."""
    self._fill(spec, rows, segments, **kwargs)
    with torch.cuda.device(self.device):
      _check(self._phase_a(self._ptrs, self._ints, self._longs, self._floats, ctypes.c_int(seg), _stream_ptr(stream)), "gar_phase_a")


_launchers = {}


def _torch_rules(spec):
  from ..aggregators import _ops
  return {"average": _ops.torch_average, "average-nan": _ops.torch_average_nan, "median": _ops.torch_median,
          "averaged-median": lambda M: _ops.torch_averaged_median(M, spec.beta), "krum": lambda M: _ops.torch_krum(M, spec.f, spec.m),
          "bulyan": lambda M: _ops.torch_bulyan(M, spec.f, spec.m), "trimmed-mean": lambda M: _ops.torch_trimmed_mean(M, spec.f),
          "mda": lambda M: _ops.torch_mda(M, spec.f), "geometric-median": lambda M: _ops.torch_geometric_median(M, spec.iterations, spec.nu)}[spec.rule]


def aggregate(spec, G, return_details=False, center=None):
  """Stand-alone aggregation of the CUDA matrix `G` ([n, d], fp32) with rule `spec` -> [d] tensor. `return_details` also returns the
  distances (Krum / Bulyan / MDA: the [n, n] matrix; geometric median, centered clipping: the [iterations, n] row distances of every
  iteration) and the selection masks. Centered clipping needs `center`, a [d] tensor of G's dtype on G's device, updated in place."""
  if not G.is_cuda:
    raise tools.UserException("ops.gar.aggregate expects a CUDA tensor")
  n, d = G.shape
  if n != spec.n:
    spec = FusedSpec(spec.rule, n, spec.f, spec.m, spec.beta, iterations=spec.iterations, nu=spec.nu, tau=spec.tau)
  if spec.rule == "centered-clipping":
    return _aggregate_centered_clipping(spec, G, return_details, center)
  if G.dtype == torch.float64 and not return_details:
    # the reference's ops are registered for double too (`native/op_krum/op.cpp:47`): the sm_90a kernels are fp32, so double inputs are
    # aggregated in double by the device-side torch implementations of the same rules (same ordering convention) instead of being rounded
    return _torch_rules(spec)(G)
  if G.dtype != torch.float32:
    out = aggregate(spec, G.float(), return_details)
    return (out[0].to(G.dtype),) + out[1:] if return_details else out.to(G.dtype)
  if n > MAX_WORKERS:  # beyond the kernels' worker limit: torch ops on the same device
    return _torch_rules(spec)(G)
  G = G.contiguous()
  pad = (-d) % 4
  if pad or G.data_ptr() % 16:
    Gp = torch.zeros((n, d + pad), dtype=G.dtype, device=G.device)
    Gp[:, :d] = G
    G = Gp
  dp = d + pad
  launcher = _launcher(G.device, n)
  out = torch.empty(dp, dtype=torch.float32, device=G.device)
  rows = [G.data_ptr() + i * dp * 4 for i in range(n)]
  launcher.launch(spec, rows, 0, dp, agg_out=out)
  out = out[:d]
  if return_details:
    dist = launcher.geo_dist_out[:spec.iterations * n].view(spec.iterations, n) if spec.rule in ITERATIVE_RULES else launcher.dist_out.view(n, n)
    return out, dist.clone(), launcher.info.clone()
  return out


def _launcher(device, n):
  key = (device.index, n)
  launcher = _launchers.get(key)
  if launcher is None:
    launcher = _launchers[key] = FusedLauncher(device, n)
  return launcher


def _aggregate_centered_clipping(spec, G, return_details, center):
  """`aggregate` for centered clipping: the sm_90a kernel for fp32 and n <= 32, the torch reference on the device otherwise."""
  from ..aggregators import _ops
  n, d = G.shape
  if center is None or center.shape != (d,) or center.device != G.device:
    raise tools.UserException("Centered clipping needs a [%d] center on %s" % (d, G.device))
  if G.dtype == torch.float64 or n > MAX_WORKERS:
    if center.dtype != G.dtype:
      raise tools.UserException("Centered clipping needs a center of type %s (got %s)" % (G.dtype, center.dtype))
    if return_details:
      raise tools.UserException("Centered clipping returns its details from the sm_90a kernel only (fp32, n <= %d)" % MAX_WORKERS)
    return _ops.torch_centered_clipping(G, spec.iterations, spec.tau, center)
  if G.dtype != torch.float32 or center.dtype != torch.float32:
    raise tools.UserException("Centered clipping on the device needs fp32 rows and center (got %s, %s)" % (G.dtype, center.dtype))
  G = G.contiguous()
  pad = (-d) % 4
  if pad or G.data_ptr() % 16:
    Gp = torch.zeros((n, d + pad), dtype=G.dtype, device=G.device)
    Gp[:, :d] = G
    G = Gp
  dp = d + pad
  work = center
  if pad or not center.is_contiguous() or center.data_ptr() % 16:
    work = torch.zeros(dp, dtype=torch.float32, device=G.device)
    work[:d] = center
  launcher = _launcher(G.device, n)
  out = torch.empty(dp, dtype=torch.float32, device=G.device)
  rows = [G.data_ptr() + i * dp * 4 for i in range(n)]
  launcher.launch(spec, rows, 0, dp, agg_out=out, center=work)
  if work is not center:
    center.copy_(work[:d])
  out = out[:d]
  if return_details:
    dist = launcher.geo_dist_out[:spec.iterations * n].view(spec.iterations, n)
    return out, dist.clone(), launcher.info.clone()
  return out


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


def craft(rows, segments, honest, byzantine, mode, coef, *, R=1, rank=0, signals=None, epoch=1, epoch_ptr=None, stream=None):
  """Craft the omniscient Byzantine rows (`attacks/omniscient.py`) over the owned `segments` of the n rows at device addresses `rows`
  (raw ints, local or peer-mapped): every slot of `byzantine` receives the ALIE / IPM value of the `honest` slots. Collective when R > 1
  (entry barrier through the signal pads, at flag value `epoch`, or `*epoch_ptr + 1` when given)."""
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
  func = _lib().agb_gar_byzantine
  func.restype = ctypes.c_int
  _check(func(c_rows, ctypes.c_int(n), lo, hi, ctypes.c_int(len(segments)), ctypes.c_uint(mask(honest)), ctypes.c_uint(mask(byzantine)),
              ctypes.c_int(BYZANTINE_MODES[mode]), ctypes.c_float(coef), ctypes.c_int(R), ctypes.c_int(rank), c_signals,
              ctypes.c_uint(epoch & 0x7fffffff), ctypes.c_ulonglong(addr(epoch_ptr)), _stream_ptr(stream)), "gar_byzantine")


def craft_byzantine_(G, byz_slots, mode, coef):
  """Stand-alone omniscient attack on the [n, d] fp32 matrix `G`, in place: rows `byz_slots` <- the ALIE (`coef` = z) or IPM
  (`coef` = epsilon) row of the other rows. CUDA tensors with n <= 32 run the sm_90a kernel; others the torch reference."""
  from ..aggregators import _ops
  n, d = G.shape
  byz_slots = _ops.check_byzantine_slots(n, byz_slots, mode)
  if not G.is_cuda or n > MAX_WORKERS:
    return _ops.torch_craft_byzantine_(G, byz_slots, mode, coef)
  if G.dtype != torch.float32:
    raise tools.UserException("ops.gar.craft_byzantine_ expects fp32 rows (got %s)" % G.dtype)
  pad = (-d) % 4
  work = G
  if pad or not G.is_contiguous() or G.data_ptr() % 16:
    work = torch.zeros((n, d + pad), dtype=G.dtype, device=G.device)
    work[:, :d] = G
  dp = d + pad
  rows = [work.data_ptr() + i * dp * 4 for i in range(n)]
  with torch.cuda.device(G.device):
    craft(rows, [(0, dp)], [i for i in range(n) if i not in byz_slots], byz_slots, mode, coef)
  if work is not G:
    index = torch.tensor(byz_slots, dtype=torch.int64, device=G.device)
    G[index] = work[index, :d]
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

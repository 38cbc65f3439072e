"""sm_90a providers of the nn ops (`native/op_nn`) — what TensorFlow's cuDNN / cuBLAS kernels are to the reference's experiments
(`experiments/cnnet.py:58-95`, `experiments/slims.py:100-125`: every layer there is a library call placed by TF).

Every function returns None (forward ops) or NotImplemented (backward ops whose legitimate result may be None) when it
does not handle the given arguments; `ops/nn.py` then either falls back to the torch provider or raises
(`AGB_NATIVE_STRICT=1`). GEMM-shaped work goes through `agb_gemm_bf16` (wgmma + TMA, `native/op_nn/gemm.cu`):

    mm_nt(x[M,K], w[N,K])  = x @ w.T      forward of dense / 1x1 conv         (A K-major,  B K-major)
    mm_nn(x[M,K], w[K,N])  = x @ w        data gradient                       (A K-major,  B MN-major)
    mm_tn(x[K,M], y[K,N])  = x.T @ y      weight gradient, split-K + fp32 red (A MN-major, B MN-major)
"""

import ctypes
import os

import torch

from . import counters

_lib_cache = None
_DISABLED = set(filter(None, os.environ.get("AGB_NATIVE_DISABLE", "").split(",")))
SM_COUNT = 132


def _lib():
  global _lib_cache
  if _lib_cache is None:
    from .. import native
    _lib_cache = native.library("op_nn")
  return _lib_cache


def _stream():
  return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
  return ctypes.c_void_p(t.data_ptr() if t is not None else 0)


def _check(status, what):
  counters.bump()
  if status != 0:
    raise RuntimeError("native op " + what + " failed with status " + str(status))


def enabled(op):
  return op not in _DISABLED and "all" not in _DISABLED


# Activation dtypes: bf16 products or fp32 (TF32 products, fp32 storage: the parity precision of the fp32 reference).
_DTYPES = (torch.bfloat16, torch.float32)


def _fn(name, tensor):
  """C entry point of a layer kernel for the element type of `tensor` (`agb_<name>` / `agb_<name>_f32`)."""
  return getattr(_lib(), name + ("_f32" if tensor.dtype == torch.float32 else ""))


# ---------------------------------------------------------------------------- #
# Pre-zeroed gradient rows: split-K weight gradients accumulate with fp32 atomics and need a zeroed destination. The trainer
# clears the whole [workers, d] gradient matrix with ONE fill before the backward pass and declares it here, which replaces
# one small fill launch per layer (53 for ResNet-50).

_prezeroed = False


class prezeroed_gradients:
  """`with prezeroed_gradients():` — destinations passed as `out=` / `grad_w` are already zero."""

  def __enter__(self):
    global _prezeroed
    self._previous, _prezeroed = _prezeroed, True

  def __exit__(self, *exc):
    global _prezeroed
    _prezeroed = self._previous
    return False


# ---------------------------------------------------------------------------- #
# Weight-gradient side stream: the weight gradient of a layer is off the critical path of the backward chain, so it can run
# next to the data gradient of the same layer (fork before, join after; under CUDA-graph capture this becomes two parallel
# branches of the graph). On for single-worker ranks (`set_launch_overlap`), AGB_WGRAD_STREAM=0|1 forces it.

_WGRAD_STREAM = os.environ.get("AGB_WGRAD_STREAM", "0") not in ("", "0")


def set_launch_overlap(flag):
  """Weight gradients on a side stream + programmatic dependent launch between the nn kernels: meant for ranks that run ONE
  batch-32 worker (small kernels, many under-filled grids), neutral-to-negative for batched workers. The trainer switches it on for single-worker ranks unless AGB_PDL /
  AGB_WGRAD_STREAM are set explicitly. Every kernel launched through `launch_pdl` must execute `griddepcontrol.wait` before touching
  global memory (`tests/test_layers_gpu.py::test_launch_overlap_keeps_gradients`)."""
  global _WGRAD_STREAM
  _WGRAD_STREAM = bool(flag)
  _lib().agb_nn_set_pdl(ctypes.c_int(1 if flag else 0))
_side_streams = {}


class _Fork:
  """`with _Fork() as fork:` runs the body on the side stream after everything issued so far on the current stream;
  `fork.join()` makes the current stream wait for it. A no-op pair when the side stream is disabled."""

  def __enter__(self):
    self.side = None
    if _WGRAD_STREAM:
      self.main = torch.cuda.current_stream()
      key = self.main.device_index
      if key not in _side_streams:
        _side_streams[key] = torch.cuda.Stream(device=self.main.device)
      self.side = _side_streams[key]
      self.side.wait_stream(self.main)
      self._ctx = torch.cuda.stream(self.side)
      self._ctx.__enter__()
    return self

  def __exit__(self, *exc):
    if self.side is not None:
      self._ctx.__exit__(*exc)
    return False

  def join(self):
    if self.side is not None:
      self.main.wait_stream(self.side)


# ---------------------------------------------------------------------------- #
# GEMM

def _rows(t, dtype=None):
  """2-D bf16 / fp32 operand with unit inner stride, row stride % 8 == 0 and a 16-byte aligned base (copy if needed)."""
  dtype = dtype if dtype is not None else (t.dtype if t.dtype in _DTYPES else torch.bfloat16)
  if t.dtype != dtype:
    t = t.to(dtype)
  if t.dim() != 2:
    t = t.reshape(t.shape[0], -1)
  if t.stride(1) == 1 and t.stride(0) % 8 == 0 and t.stride(0) >= t.shape[1] and t.data_ptr() % 16 == 0:
    return t
  rows, cols = t.shape
  ld = (cols + 7) // 8 * 8
  buf = torch.zeros((rows, ld), dtype=dtype, device=t.device)
  buf[:, :cols] = t
  return buf[:, :cols]


def set_gemm_persistent(enabled):
  """Launch the GEMM persistently (one CTA per SM walking the tiles) or with one CTA per tile."""
  _lib().agb_gemm_set_persistent(ctypes.c_int(1 if enabled else 0))


def alloc_out(m, n, dtype, device):
  """[m, n] view of a buffer whose row stride is a multiple of 8 elements (so it can feed the next GEMM through TMA)."""
  ld = (n + 7) // 8 * 8
  return torch.empty((m, ld), dtype=dtype, device=device)[:, :n]


def _gemm(a, b, out, M, N, K, a_mn, b_mn, bias, relu, splits, bn, groups=1, group_stride=0):
  if out.stride(1) != 1:
    raise RuntimeError("GEMM output must have unit inner stride")
  if a.dtype == torch.float32:   # TF32 products, fp32 output
    if b.dtype != torch.float32 or out.dtype != torch.float32:
      raise RuntimeError("TF32 GEMM needs fp32 operands and output")
    status = _lib().agb_gemm_tf32_grouped(_ptr(a), _ptr(b), _ptr(out), ctypes.c_int(M), ctypes.c_int(N), ctypes.c_int(K), ctypes.c_longlong(a.stride(0)), ctypes.c_longlong(b.stride(0)),
                                          ctypes.c_longlong(out.stride(0)), ctypes.c_int(1 if a_mn else 0), ctypes.c_int(1 if b_mn else 0), _ptr(bias), ctypes.c_int(1 if relu else 0),
                                          ctypes.c_int(splits), ctypes.c_int(128 if bn == 256 else bn), ctypes.c_int(groups), ctypes.c_longlong(group_stride), _stream())
    _check(status, "gemm_tf32")
    return out
  func = _lib().agb_gemm_bf16_grouped
  out_fp32 = 1 if out.dtype == torch.float32 else 0
  status = func(_ptr(a), _ptr(b), _ptr(out), ctypes.c_int(M), ctypes.c_int(N), ctypes.c_int(K), ctypes.c_longlong(a.stride(0)), ctypes.c_longlong(b.stride(0)),
                ctypes.c_longlong(out.stride(0)), ctypes.c_int(1 if a_mn else 0), ctypes.c_int(1 if b_mn else 0), _ptr(bias), ctypes.c_int(1 if relu else 0),
                ctypes.c_int(out_fp32), ctypes.c_int(splits), ctypes.c_int(bn), ctypes.c_int(groups), ctypes.c_longlong(group_stride), _stream())
  _check(status, "gemm_bf16")
  return out


def mm_nt(x, w, bias=None, relu=False, out=None, out_dtype=None, bn=0):
  """x[M,K] @ w[N,K]^T (+ fp32 bias[N], ReLU). fp32 operands are multiplied as TF32."""
  x = _rows(x)
  w = _rows(w, x.dtype)
  M, K = x.shape
  N = w.shape[0]
  if out is None:
    out = alloc_out(M, N, (out_dtype or x.dtype) if x.dtype == torch.bfloat16 else torch.float32, x.device)
  if bias is not None and bias.dtype != torch.float32:
    bias = bias.float()
  return _gemm(x, w, out, M, N, K, False, False, bias, relu, 1, bn)


def mm_nn(x, w, out=None, out_dtype=None, bn=0):
  """x[M,K] @ w[K,N]."""
  x = _rows(x)
  w = _rows(w, x.dtype)
  M, K = x.shape
  N = w.shape[1]
  if out is None:
    out = alloc_out(M, N, (out_dtype or x.dtype) if x.dtype == torch.bfloat16 else torch.float32, x.device)
  return _gemm(x, w, out, M, N, K, False, True, None, False, 1, bn)


# Split-K weight gradients accumulate their partial products with fp32 reductions (red.global.add.v4.f32) whose arrival order varies
# from run to run: the last bits of a gradient can differ between two executions of the same step. `AGB_DETERMINISTIC=1` /
# `set_deterministic(True)` gives bit-reproducible gradients by keeping every weight-gradient product in ONE accumulation chain per
# output tile (no split-K): each tile is then summed in registers in a fixed k order. Slower on layers with few output tiles.
_DETERMINISTIC = os.environ.get("AGB_DETERMINISTIC", "0") not in ("", "0")


def set_deterministic(flag):
  global _DETERMINISTIC
  _DETERMINISTIC = bool(flag)


def pick_splits(m_out, n_out, k, bn=128):
  if _DETERMINISTIC:
    return 1
  tiles = ((m_out + 127) // 128) * ((n_out + bn - 1) // bn)
  kblocks = (k + 63) // 64
  want = max(1, (2 * SM_COUNT + tiles - 1) // tiles)
  return max(1, min(kblocks, want, 128))


def _all_groups(out, groups, group_stride):
  """[groups, *out.shape] strided view over every logical worker's copy of `out` (worker 0's view of the gradient matrix)."""
  if groups == 1:
    return out
  return out.as_strided((groups,) + tuple(out.shape), (group_stride,) + tuple(out.stride()), out.storage_offset())


def mm_tn(x, y, out=None, splits=None, bn=0, groups=1, group_stride=0):
  """x[K,M]^T @ y[K,N] -> fp32 [M,N]; split-K partial sums are accumulated with fp32 atomics (out is zeroed here).
  `groups` > 1: x and y hold `groups` consecutive blocks of K / groups rows, one product per block, written `group_stride`
  elements apart starting at `out` (the per-worker weight gradients, one launch)."""
  x = _rows(x)
  y = _rows(y, x.dtype)
  K, M = x.shape
  N = y.shape[1]
  if groups > 1:
    if K % groups or y.shape[0] != K:
      raise ValueError("mm_tn: %d and %d rows do not split into %d equal groups" % (K, y.shape[0], groups))
    # every group needs its own output: with a shared one the groups' products would be summed (split-K) or race
    if out is None or group_stride < (M - 1) * out.stride(0) + N:
      raise ValueError("mm_tn: %d groups need an out= and a group_stride of at least one [%d, %d] output, got %s" % (groups, M, N, group_stride))
  K //= groups
  fresh = out is None
  if fresh:
    out = torch.empty((M, N), dtype=torch.float32, device=x.device)
  if splits is None:
    splits = max(1, pick_splits(M, N, K, 64 if N <= 64 else 128) // groups)
  if splits > 1 and (fresh or not _prezeroed):
    _all_groups(out, groups, group_stride).zero_()
  return _gemm(x, y, out, M, N, K, True, True, None, False, splits, bn, groups, group_stride)


# ---------------------------------------------------------------------------- #
# Dense

def _masked(dy, y, relu):
  if not relu:
    return dy
  out = relu_backward(dy, y)
  return out if out is not None else dy * (y > 0).to(dy.dtype)


def linear_forward(x, weight, bias, relu):
  if not enabled("linear"):
    return None
  return mm_nt(x, weight, bias, relu)


def linear_backward(dy, x, weight, y, relu, need_dx, grad_w, grad_b, groups=1, group_stride=0):
  if not enabled("linear"):
    return NotImplemented
  dy = _rows(_masked(dy, y, relu))
  with _Fork() as fork:
    mm_tn(dy, x, out=grad_w, groups=groups, group_stride=group_stride)
    if grad_b is not None:
      colsum(dy, out=grad_b, groups=groups, group_stride=group_stride)
  dx = mm_nn(dy, weight) if need_dx else None
  fork.join()
  return dx


# ---------------------------------------------------------------------------- #
# Convolution (1x1 stride-1 convolutions are GEMMs on the NHWC view; other shapes: see conv.py when available)

def _as_rows(x):
  """(N, C, H, W) channels_last -> [N*H*W, C] view."""
  n, c, h, w = x.shape
  return x.permute(0, 2, 3, 1).reshape(n * h * w, c)


def _from_rows(y2d, n, h, w):
  return y2d.view(n, h, w, y2d.shape[1]).permute(0, 3, 1, 2)


def _is_pointwise(weight, stride, pads):
  return weight.shape[1] == 1 and weight.shape[2] == 1 and stride == 1 and not any(pads)


def conv2d_forward(x, weight, bias, stride, pads, relu, aux=None):
  """`aux`: optional dict that lives until the matching backward call; the im2col path leaves its column matrix there."""
  if not enabled("conv"):
    return None
  if _is_pointwise(weight, stride, pads) and x.is_contiguous(memory_format=torch.channels_last) and x.shape[1] % 8 == 0:
    n, c, h, w = x.shape
    y = mm_nt(_as_rows(x), weight.reshape(weight.shape[0], -1), bias, relu)
    return _from_rows(y if y.stride(0) == y.shape[1] else y.contiguous(), n, h, w)
  if _implicit_ok(x, weight, stride, pads):
    return conv2d_forward_implicit(x, weight, bias, relu, stride, pads)
  if enabled("convk") and _general_ok(x, weight):
    return conv2d_forward_general(x, weight, bias, stride, pads, relu, aux)
  return None


def conv2d_backward(dy, x, weight, y, stride, pads, relu, has_bias, need_dx, grad_w, grad_b, groups=1, group_stride=0, aux=None):
  if not enabled("conv"):
    return NotImplemented
  if _is_pointwise(weight, stride, pads) and x.is_contiguous(memory_format=torch.channels_last) and x.shape[1] % 8 == 0 and weight.shape[0] % 8 == 0:
    n, c, h, w = x.shape
    dy = _masked(dy, y, relu)
    if not dy.is_contiguous(memory_format=torch.channels_last):
      dy = dy.contiguous(memory_format=torch.channels_last)
    dy2d = _as_rows(dy)
    with _Fork() as fork:
      mm_tn(dy2d, _as_rows(x), out=grad_w.view(grad_w.shape[0], -1), groups=groups, group_stride=group_stride)
      if has_bias:
        colsum(dy2d, out=grad_b, groups=groups, group_stride=group_stride)
    dx = _from_rows(mm_nn(dy2d, weight.reshape(weight.shape[0], -1)), n, h, w) if need_dx else None
    fork.join()
    return dx
  if _implicit_ok(x, weight, stride, pads) and dy.dtype == x.dtype:
    return conv2d_backward_implicit(dy, x, weight, y, relu, has_bias, need_dx, grad_w, grad_b, groups, group_stride, stride, pads)
  if enabled("convk") and _general_ok(x, weight) and dy.dtype == x.dtype:
    return conv2d_backward_general(dy, x, weight, y, stride, pads, relu, has_bias, need_dx, grad_w, grad_b, groups, group_stride, aux)
  return NotImplemented


# ---------------------------------------------------------------------------- #
# General k x k convolution: im2col (bf16, column order kh, kw, c) + the same three GEMMs

def _im2col(x, kh, kw, stride, pads, oh, ow):
  n, c, h, w = x.shape
  kcol = kh * kw * c
  ld = (kcol + 7) // 8 * 8
  col = torch.empty((n * oh * ow, ld), dtype=x.dtype, device=x.device)
  func = _fn("agb_im2col", x)
  _check(func(_ptr(x), _ptr(col), ctypes.c_int(n), ctypes.c_int(h), ctypes.c_int(w), ctypes.c_int(c), ctypes.c_int(oh), ctypes.c_int(ow), ctypes.c_int(kh), ctypes.c_int(kw),
              ctypes.c_int(stride), ctypes.c_int(pads[0]), ctypes.c_int(pads[2]), ctypes.c_longlong(ld), _stream()), "im2col")
  return col[:, :kcol]


def _out_size(size, k, stride, lo, hi):
  return (size + lo + hi - k) // stride + 1


def _weight_rows(weight):
  """[Cout, kh, kw, Cin] -> [Cout, kh*kw*Cin] rows with a TMA-compatible stride (copy only for the 3-channel stem)."""
  return weight.reshape(weight.shape[0], -1)


def _general_ok(x, weight):
  return x.is_contiguous(memory_format=torch.channels_last) and x.dtype in _DTYPES and weight.shape[0] % 8 == 0


def conv2d_forward_general(x, weight, bias, stride, pads, relu, aux=None):
  n, c, h, w = x.shape
  kh, kw = weight.shape[1], weight.shape[2]   # rectangular filters too (the 1x7 / 7x1 / 1x3 / 3x1 factorised kernels of the Inception families)
  oh, ow = _out_size(h, kh, stride, pads[0], pads[1]), _out_size(w, kw, stride, pads[2], pads[3])
  col = _im2col(x, kh, kw, stride, pads, oh, ow)
  if aux is not None:
    aux["col"] = col  # the weight gradient multiplies by the same matrix: keep it instead of rebuilding it
  y = mm_nt(col, _weight_rows(weight), bias, relu)
  return _from_rows(y if y.stride(0) == y.shape[1] else y.contiguous(), n, oh, ow)


def conv2d_backward_general(dy, x, weight, y, stride, pads, relu, has_bias, need_dx, grad_w, grad_b, groups=1, group_stride=0, aux=None):
  n, c, h, w = x.shape
  kh, kw = weight.shape[1], weight.shape[2]
  oh, ow = dy.shape[2], dy.shape[3]
  dy = _masked(dy, y, relu)
  if not dy.is_contiguous(memory_format=torch.channels_last):
    dy = dy.contiguous(memory_format=torch.channels_last)
  dy2d = _as_rows(dy)
  if need_dx and c % 8:
    return NotImplemented
  col = aux.pop("col", None) if aux is not None else None
  if col is None or col.shape[0] != n * oh * ow:
    col = _im2col(x, kh, kw, stride, pads, oh, ow)
  with _Fork() as fork:
    mm_tn(dy2d, col, out=grad_w.view(grad_w.shape[0], -1), groups=groups, group_stride=group_stride)
    if has_bias:
      colsum(dy2d, out=grad_b, groups=groups, group_stride=group_stride)
  if not need_dx:
    fork.join()
    return None
  dcol = mm_nn(dy2d, _weight_rows(weight))
  dx = torch.empty((n, h, w, c), dtype=x.dtype, device=x.device)
  func = _fn("agb_col2im", x)
  _check(func(_ptr(dcol), _ptr(dx), ctypes.c_int(n), ctypes.c_int(h), ctypes.c_int(w), ctypes.c_int(c), ctypes.c_int(oh), ctypes.c_int(ow), ctypes.c_int(kh), ctypes.c_int(kw),
              ctypes.c_int(stride), ctypes.c_int(pads[0]), ctypes.c_int(pads[2]), ctypes.c_longlong(dcol.stride(0)), _stream()), "col2im")
  fork.join()
  return dx.permute(0, 3, 1, 2)


# ---------------------------------------------------------------------------- #
# Implicit-GEMM convolution (native/op_nn/conv.cu): Cin % 64 == 0, Cout % 64 == 0, square k x k filters;
#   stride 1: odd k, "same" padding (output grid = input grid);
#   stride 2: even H and W, output H/2 x W/2 (slim `conv2d_same`'s explicit (k-1)//2 padding, or TF "SAME"), k >= 2.

def _implicit_geometry(x, weight, stride, pads):
  """(OH, OW) when the implicit-GEMM kernels take this convolution, else None."""
  k = weight.shape[1]
  chunk = 64 if x.dtype == torch.bfloat16 else 32   # channels per 128-byte swizzle row
  if not (enabled("implicit") and k > 1 and weight.shape[2] == k and x.shape[1] % chunk == 0 and weight.shape[0] % chunk == 0 and x.dtype in _DTYPES and weight.dtype == x.dtype
          and x.is_contiguous(memory_format=torch.channels_last) and weight.is_contiguous()):
    return None
  h, w = x.shape[2], x.shape[3]
  oh, ow = _out_size(h, k, stride, pads[0], pads[1]), _out_size(w, k, stride, pads[2], pads[3])
  if stride == 1:
    pad = (k - 1) // 2
    return (oh, ow) if (k % 2 == 1 and tuple(pads) == (pad, pad, pad, pad)) else None
  if stride == 2 and enabled("implicit2") and h % 2 == 0 and w % 2 == 0 and (oh, ow) == (h // 2, w // 2) and pads[0] < k and pads[2] < k:
    return oh, ow
  return None


def _implicit_ok(x, weight, stride, pads):
  return _implicit_geometry(x, weight, stride, pads) is not None


def _conv_implicit(mode, act, other, out, n, h, w, oh, ow, cin, cout, k, stride, pads, bias=None, relu=False, splits=1, bn=0, groups=1, group_stride=0):
  if act.dtype == torch.float32:   # TF32 products
    _check(_lib().agb_conv_implicit_strided_tf32(ctypes.c_int(mode), _ptr(act), _ptr(other), _ptr(out), ctypes.c_int(n), ctypes.c_int(h), ctypes.c_int(w), ctypes.c_int(oh), ctypes.c_int(ow),
                                                 ctypes.c_int(cin), ctypes.c_int(cout), ctypes.c_int(k), ctypes.c_int(stride), ctypes.c_int(pads[0]), ctypes.c_int(pads[2]), _ptr(bias),
                                                 ctypes.c_int(1 if relu else 0), ctypes.c_int(splits), ctypes.c_int(bn), ctypes.c_int(groups), ctypes.c_longlong(group_stride), _stream()),
           "conv_implicit_tf32")
    return out
  _check(_lib().agb_conv_implicit_strided(ctypes.c_int(mode), _ptr(act), _ptr(other), _ptr(out), ctypes.c_int(n), ctypes.c_int(h), ctypes.c_int(w), ctypes.c_int(oh), ctypes.c_int(ow),
                                          ctypes.c_int(cin), ctypes.c_int(cout), ctypes.c_int(k), ctypes.c_int(stride), ctypes.c_int(pads[0]), ctypes.c_int(pads[2]), _ptr(bias),
                                          ctypes.c_int(1 if relu else 0), ctypes.c_int(1 if out.dtype == torch.float32 else 0), ctypes.c_int(splits), ctypes.c_int(bn), ctypes.c_int(groups),
                                          ctypes.c_longlong(group_stride), _stream()), "conv_implicit")
  return out


def conv2d_forward_implicit(x, weight, bias, relu, stride=1, pads=None):
  n, cin, h, w = x.shape
  cout, k = weight.shape[0], weight.shape[1]
  pads = pads if pads is not None else ((k - 1) // 2,) * 4
  oh, ow = _implicit_geometry(x, weight, stride, pads)
  y = torch.empty((n, oh, ow, cout), dtype=x.dtype, device=x.device)
  if bias is not None and bias.dtype != torch.float32:
    bias = bias.float()
  _conv_implicit(0, x, weight, y, n, h, w, oh, ow, cin, cout, k, stride, pads, bias, relu)
  return y.permute(0, 3, 1, 2)


def conv2d_backward_implicit(dy, x, weight, y, relu, has_bias, need_dx, grad_w, grad_b, groups=1, group_stride=0, stride=1, pads=None):
  n, cin, h, w = x.shape
  cout, k = weight.shape[0], weight.shape[1]
  pads = pads if pads is not None else ((k - 1) // 2,) * 4
  oh, ow = dy.shape[2], dy.shape[3]
  dy = _masked(dy, y, relu)
  if not dy.is_contiguous(memory_format=torch.channels_last):
    dy = dy.contiguous(memory_format=torch.channels_last)
  tiles = k * k * ((cout + 127) // 128) * ((cin + 127) // 128)
  kblocks = max(1, n * oh * ow // (64 if x.dtype == torch.bfloat16 else 32) // groups)
  splits = 1 if _DETERMINISTIC else max(1, min(kblocks, (2 * SM_COUNT + tiles * groups - 1) // (tiles * groups), 64))
  with _Fork() as fork:
    if not _prezeroed:
      _all_groups(grad_w, groups, group_stride).zero_()
    _conv_implicit(2, dy, x, grad_w, n, h, w, oh, ow, cin, cout, k, stride, pads, splits=splits, groups=groups, group_stride=group_stride)
    if has_bias:
      colsum(_as_rows(dy), out=grad_b, groups=groups, group_stride=group_stride)
  dx = None
  if need_dx:
    dx = torch.empty((n, h, w, cin), dtype=x.dtype, device=x.device)
    _conv_implicit(1, dy, weight, dx, n, h, w, oh, ow, cin, cout, k, stride, pads)
    dx = dx.permute(0, 3, 1, 2)
  fork.join()
  return dx


# ---------------------------------------------------------------------------- #
# Memory-bound layers (native/op_nn/layers.cu)

_workspaces = {}


def _workspace(device, name, numel, dtype):
  key = (device, name, dtype)
  buf = _workspaces.get(key)
  if buf is None or buf.numel() < numel:
    buf = _workspaces[key] = torch.zeros(max(numel, 4096), dtype=dtype, device=device)   # statistics kernels expect (and leave) zeros
  return buf


def _cl_ok(*tensors, dtypes=_DTYPES):
  """Every given tensor is channels_last (when 4-D) and they all share one supported activation dtype."""
  present = [t for t in tensors if t is not None]
  if not present or present[0].dtype not in dtypes or any(t.dtype != present[0].dtype for t in present):
    return False
  return all(t.dim() != 4 or t.is_contiguous(memory_format=torch.channels_last) for t in present)


def colsum(dy2d, y2d=None, out=None, groups=1, group_stride=0):
  """fp32 column sums of a [rows, C] bf16 matrix (optionally masked by y > 0): bias gradients. With `groups` > 1 one sum per
  consecutive block of rows, written `group_stride` elements apart starting at `out`."""
  rows, c = dy2d.shape
  if out is None:
    out = torch.empty(c, dtype=torch.float32, device=dy2d.device)
  if c % 8 or dy2d.stride(0) != c:
    src = dy2d.float() if y2d is None else dy2d.float() * (y2d > 0)
    _all_groups(out, groups, group_stride).copy_(src.reshape(groups, rows // groups, c).sum(dim=1) if groups > 1 else src.sum(dim=0))
    return out
  sums = _workspace(dy2d.device, "colsum", 2 * c * groups + 1, torch.float64)
  _check(_fn("agb_colsum", dy2d)(_ptr(dy2d), _ptr(y2d), _ptr(out), _ptr(sums), ctypes.c_longlong(rows), ctypes.c_int(c), ctypes.c_int(groups), ctypes.c_longlong(group_stride), _stream()), "colsum")
  return out


_BN_FUSED = os.environ.get("AGB_BN_FUSED", "1") not in ("", "0")
_BN_UNSUPPORTED = 399


def set_bn_fused(flag):
  """Select the single-launch (resident-tile) batch-norm kernels or the statistics + apply pair."""
  global _BN_FUSED
  _BN_FUSED = bool(flag)


def set_bn_fused_limits(forward_mb=72, backward_mb=40, min_rows=4096):
  """Envelope of the single-launch kernels: largest tensor (MB) per direction and fewest rows (defaults: `g_fused_max_mb` / `g_fused_min_rows` of `native/op_nn/layers.cu`)."""
  _lib().agb_bn_fused_set_limits(ctypes.c_longlong(forward_mb), ctypes.c_longlong(backward_mb), ctypes.c_longlong(min_rows))


def _bn_fused_workspace(device, name):
  lib = _lib()
  lib.agb_bn_fused_workspace_bytes.restype = ctypes.c_longlong
  return _workspace(device, name, int(lib.agb_bn_fused_workspace_bytes()), torch.uint8)


def batchnorm_forward(x, gamma, beta, moving_mean, moving_var, decay, eps, relu, groups=1, residual=None):
  """`residual`: y = relu?(bn(x) + residual), only through the single-launch kernel (None when it cannot take the shape)."""
  if not enabled("bn") or not _cl_ok(x, residual) or x.shape[1] % 8:
    return None
  n, c, h, w = x.shape
  rows = n * h * w
  if residual is not None and (residual.shape != x.shape or not residual.is_contiguous(memory_format=torch.channels_last)):
    return None
  y = torch.empty_like(x, memory_format=torch.channels_last)
  stats = torch.empty((4, groups * c), dtype=torch.float32, device=x.device)  # save_mean, save_rstd, scale, shift
  if _BN_FUSED and x.dtype == torch.bfloat16:   # the resident-tile kernel is sized for 2-byte activations
    status = _lib().agb_bn_forward_fused(_ptr(x), _ptr(residual), _ptr(y), _ptr(gamma), _ptr(beta), _ptr(moving_mean), _ptr(moving_var), _ptr(stats[0]), _ptr(stats[1]),
                                         _ptr(_bn_fused_workspace(x.device, "bn_fused_fwd")), ctypes.c_longlong(rows), ctypes.c_int(c), ctypes.c_int(groups),
                                         ctypes.c_float(eps), ctypes.c_float(decay), ctypes.c_int(1 if relu else 0), _stream())
    if status != _BN_UNSUPPORTED:
      _check(status, "bn_forward_fused")
      return y, stats[0], stats[1]
  sums = _workspace(x.device, "bn_sums", 2 * groups * c + 1, torch.float64)
  _check(_fn("agb_bn_forward", x)(_ptr(x), _ptr(residual), _ptr(y), _ptr(gamma), _ptr(beta), _ptr(moving_mean), _ptr(moving_var), _ptr(stats[0]), _ptr(stats[1]), _ptr(sums),
                               _ptr(stats[2]), _ptr(stats[3]), ctypes.c_longlong(rows), ctypes.c_int(c), ctypes.c_int(groups), ctypes.c_float(eps),
                               ctypes.c_float(decay), ctypes.c_int(1 if relu else 0), _stream()), "bn_forward")
  return y, stats[0], stats[1]


def batchnorm_backward(dy, x, y, gamma, mean, rstd, relu, grad_gamma, grad_beta, groups=1, group_stride=0, want_masked=False):
  """`want_masked` (needs `relu`): returns (dx, dy * (y > 0)) — single-launch kernel only (None when it cannot take the shape)."""
  if not enabled("bn") or not _cl_ok(x, dy, y) or x.shape[1] % 8 or (want_masked and not relu):
    return None
  if not dy.is_contiguous(memory_format=torch.channels_last):
    dy = dy.contiguous(memory_format=torch.channels_last)
  n, c, h, w = x.shape
  rows = n * h * w
  dx = torch.empty_like(x, memory_format=torch.channels_last)
  masked = torch.empty_like(dy, memory_format=torch.channels_last) if want_masked else None
  if _BN_FUSED and x.dtype == torch.bfloat16:
    status = _lib().agb_bn_backward_fused(_ptr(dy), _ptr(x), _ptr(y if relu else None), _ptr(gamma), _ptr(mean), _ptr(rstd), _ptr(dx), _ptr(masked), _ptr(grad_gamma),
                                          _ptr(grad_beta), _ptr(_bn_fused_workspace(x.device, "bn_fused_bwd")), ctypes.c_longlong(rows), ctypes.c_int(c), ctypes.c_int(groups),
                                          ctypes.c_longlong(group_stride), _stream())
    if status != _BN_UNSUPPORTED:
      _check(status, "bn_backward_fused")
      return (dx, masked) if want_masked else dx
  sums = _workspace(x.device, "bn_sums", 2 * groups * c + 1, torch.float64)
  coef = _workspace(x.device, "bn_coef", 3 * groups * c, torch.float32)
  _check(_fn("agb_bn_backward", x)(_ptr(dy), _ptr(x), _ptr(y if relu else None), _ptr(gamma), _ptr(mean), _ptr(rstd), _ptr(dx), _ptr(masked), _ptr(grad_gamma), _ptr(grad_beta),
                                _ptr(sums), _ptr(coef), ctypes.c_longlong(rows), ctypes.c_int(c), ctypes.c_int(groups), ctypes.c_longlong(group_stride), _stream()), "bn_backward")
  return (dx, masked) if want_masked else dx


def layernorm_forward(x, gamma, beta, eps):
  if not enabled("layernorm") or x.dtype != torch.bfloat16 or x.dim() != 2 or not x.is_contiguous() or x.shape[1] % 8 or x.shape[1] > 5632:
    return None
  rows, c = x.shape
  y = torch.empty_like(x)
  mean = torch.empty(rows, dtype=torch.float32, device=x.device)
  rstd = torch.empty(rows, dtype=torch.float32, device=x.device)
  _check(_lib().agb_layernorm_forward(_ptr(x), _ptr(y), _ptr(gamma), _ptr(beta), _ptr(mean), _ptr(rstd), ctypes.c_longlong(rows), ctypes.c_int(c), ctypes.c_float(eps), _stream()), "layernorm_forward")
  return y, mean, rstd


def layernorm_backward(dy, x, gamma, mean, rstd, grad_gamma, grad_beta):
  if not enabled("layernorm") or x.dtype != torch.bfloat16 or x.dim() != 2 or not x.is_contiguous() or x.shape[1] % 8 or x.shape[1] > 5632:
    return None
  dy = dy.contiguous()
  rows, c = x.shape
  dx = torch.empty_like(x)
  grad_gamma.zero_()
  grad_beta.zero_()
  _check(_lib().agb_layernorm_backward(_ptr(dy), _ptr(x), _ptr(gamma), _ptr(mean), _ptr(rstd), _ptr(dx), _ptr(grad_gamma), _ptr(grad_beta), ctypes.c_longlong(rows), ctypes.c_int(c), _stream()), "layernorm_backward")
  return dx


# ---------------------------------------------------------------------------- #
# Depthwise convolution, SAME average pooling, ReLU6 (native/op_nn/depthwise.cu): on by default; `AGB_NATIVE_DEPTHWISE=0` routes these layers to the aten provider.

_DEPTHWISE = os.environ.get("AGB_NATIVE_DEPTHWISE", os.environ.get("AGB_NATIVE_PREVIEW", "1")) not in ("", "0")


def _depthwise_ok(x, weight):
  return (_DEPTHWISE and enabled("depthwise") and _cl_ok(x, dtypes=(torch.bfloat16,)) and x.dim() == 4 and x.shape[1] % 8 == 0 and weight.shape[0] == x.shape[1] and weight.shape[1] == weight.shape[2]
          and weight.dtype == torch.bfloat16)


def _transposed_taps(weight):
  """[C, k, k, 1] bf16 -> [k*k, C]: the 8 channels of a thread become one 16-byte load per tap."""
  c, k = weight.shape[0], weight.shape[1]
  return weight.reshape(c, k * k).t().contiguous()


def depthwise_forward(x, weight, stride, pads):
  if not _depthwise_ok(x, weight):
    return None
  n, c, h, w = x.shape
  k = weight.shape[1]
  oh, ow = _out_size(h, k, stride, pads[0], pads[1]), _out_size(w, k, stride, pads[2], pads[3])
  y = torch.empty((n, oh, ow, c), dtype=torch.bfloat16, device=x.device)
  _check(_lib().agb_depthwise_forward(_ptr(x), _ptr(_transposed_taps(weight)), _ptr(y), ctypes.c_int(n), ctypes.c_int(h), ctypes.c_int(w), ctypes.c_int(c), ctypes.c_int(oh),
                                      ctypes.c_int(ow), ctypes.c_int(k), ctypes.c_int(stride), ctypes.c_int(pads[0]), ctypes.c_int(pads[2]), _stream()), "depthwise_forward")
  return y.permute(0, 3, 1, 2)


def depthwise_backward(dy, x, weight, stride, pads, grad_w, groups=1, group_stride=0):
  """Returns dx; writes the per-worker weight gradients into `grad_w` ([C, k, k, 1] fp32 view of worker 0's row)."""
  if not _depthwise_ok(x, weight) or dy.dtype != torch.bfloat16:
    return None
  if not dy.is_contiguous(memory_format=torch.channels_last):
    dy = dy.contiguous(memory_format=torch.channels_last)
  n, c, h, w = x.shape
  k = weight.shape[1]
  oh, ow = dy.shape[2], dy.shape[3]
  geometry = (ctypes.c_int(n), ctypes.c_int(h), ctypes.c_int(w), ctypes.c_int(c), ctypes.c_int(oh), ctypes.c_int(ow), ctypes.c_int(k), ctypes.c_int(stride),
              ctypes.c_int(pads[0]), ctypes.c_int(pads[2]))
  if not _prezeroed:
    _all_groups(grad_w, groups, group_stride).zero_()
  _check(_lib().agb_depthwise_wgrad(_ptr(dy), _ptr(x), _ptr(grad_w), *geometry, ctypes.c_int(groups), ctypes.c_longlong(group_stride), _stream()), "depthwise_wgrad")
  dx = torch.empty((n, h, w, c), dtype=torch.bfloat16, device=x.device)
  _check(_lib().agb_depthwise_dgrad(_ptr(dy), _ptr(_transposed_taps(weight)), _ptr(dx), *geometry, _stream()), "depthwise_dgrad")
  return dx.permute(0, 3, 1, 2)


def avgpool2d_forward(x, k, stride, pads):
  if not (_DEPTHWISE and enabled("pool") and _cl_ok(x, dtypes=(torch.bfloat16,)) and x.dim() == 4 and x.shape[1] % 8 == 0):
    return None
  n, c, h, w = x.shape
  oh, ow = _out_size(h, k, stride, pads[0], pads[1]), _out_size(w, k, stride, pads[2], pads[3])
  y = torch.empty((n, oh, ow, c), dtype=torch.bfloat16, device=x.device)
  _check(_lib().agb_avgpool2d_forward(_ptr(x), _ptr(y), ctypes.c_int(n), ctypes.c_int(h), ctypes.c_int(w), ctypes.c_int(c), ctypes.c_int(oh), ctypes.c_int(ow), ctypes.c_int(k),
                                      ctypes.c_int(stride), ctypes.c_int(pads[0]), ctypes.c_int(pads[2]), _stream()), "avgpool2d_forward")
  return y.permute(0, 3, 1, 2)


def avgpool2d_backward(dy, shape, k, stride, pads):
  n, c, h, w = shape
  if not (_DEPTHWISE and enabled("pool") and _cl_ok(dy, dtypes=(torch.bfloat16,)) and dy.dim() == 4 and c % 8 == 0):
    return None
  if not dy.is_contiguous(memory_format=torch.channels_last):
    dy = dy.contiguous(memory_format=torch.channels_last)
  dx = torch.empty((n, h, w, c), dtype=torch.bfloat16, device=dy.device)
  _check(_lib().agb_avgpool2d_backward(_ptr(dy), _ptr(dx), ctypes.c_int(n), ctypes.c_int(h), ctypes.c_int(w), ctypes.c_int(c), ctypes.c_int(dy.shape[2]), ctypes.c_int(dy.shape[3]),
                                       ctypes.c_int(k), ctypes.c_int(stride), ctypes.c_int(pads[0]), ctypes.c_int(pads[2]), _stream()), "avgpool2d_backward")
  return dx.permute(0, 3, 1, 2)


def relu6(x, dy=None):
  """Forward clamp (dy None) or backward mask of ReLU6."""
  tensors = (x,) if dy is None else (x, dy)
  if not (_DEPTHWISE and enabled("eltwise")) or any(t.dtype != torch.bfloat16 or t.numel() % 8 for t in tensors):
    return None
  if dy is not None and (dy.stride() != x.stride() or dy.shape != x.shape):
    return None
  if not (x.is_contiguous() or x.is_contiguous(memory_format=torch.channels_last)):
    return None
  out = torch.empty_like(x)
  _check(_lib().agb_relu6(_ptr(x), _ptr(dy), _ptr(out), ctypes.c_longlong(x.numel()), _stream()), "relu6")
  return out


def subsample_forward(x, stride):
  if not enabled("eltwise") or not _cl_ok(x) or x.dim() != 4 or x.shape[1] % 8:
    return None
  n, c, h, w = x.shape
  y = torch.empty((n, -(-h // stride), -(-w // stride), c), dtype=x.dtype, device=x.device)
  status = _fn("agb_subsample_forward", x)(_ptr(x), _ptr(y), ctypes.c_int(n), ctypes.c_int(h), ctypes.c_int(w), ctypes.c_int(c), ctypes.c_int(stride), _stream())
  if status == _BN_UNSUPPORTED:
    return None
  _check(status, "subsample_forward")
  return y.permute(0, 3, 1, 2)


def subsample_backward(dy, shape, stride):
  n, c, h, w = shape
  if not enabled("eltwise") or not _cl_ok(dy) or dy.dim() != 4 or c % 8:
    return None
  if not dy.is_contiguous(memory_format=torch.channels_last):
    dy = dy.contiguous(memory_format=torch.channels_last)
  dx = torch.empty((n, h, w, c), dtype=dy.dtype, device=dy.device)
  status = _fn("agb_subsample_backward", dy)(_ptr(dy), _ptr(dx), ctypes.c_int(n), ctypes.c_int(h), ctypes.c_int(w), ctypes.c_int(c), ctypes.c_int(stride), _stream())
  if status == _BN_UNSUPPORTED:
    return None
  _check(status, "subsample_backward")
  return dx.permute(0, 3, 1, 2)


def relu_backward(dy, y):
  if not enabled("eltwise") or dy.dtype not in _DTYPES or y.dtype != dy.dtype or dy.numel() % 8 or dy.stride() != y.stride() or not (dy.is_contiguous() or dy.is_contiguous(memory_format=torch.channels_last)):
    return None
  dx = torch.empty_like(dy)
  _check(_fn("agb_relu_backward", dy)(_ptr(dy), _ptr(y), _ptr(dx), ctypes.c_longlong(dy.numel()), _stream()), "relu_backward")
  return dx


def add_relu_forward(a, b, relu):
  if not enabled("eltwise") or a.dtype not in _DTYPES or b.dtype != a.dtype or a.numel() % 8 or a.stride() != b.stride() or not (a.is_contiguous() or a.is_contiguous(memory_format=torch.channels_last)):
    return None
  out = torch.empty_like(a)
  _check(_fn("agb_add_relu", a)(_ptr(a), _ptr(b), _ptr(out), ctypes.c_longlong(a.numel()), ctypes.c_int(1 if relu else 0), _stream()), "add_relu")
  return out


def maxpool_forward(x, k, stride, pads):
  if not enabled("pool") or not _cl_ok(x) or x.shape[1] % 8:
    return None
  n, c, h, w = x.shape
  oh, ow = _out_size(h, k, stride, pads[0], pads[1]), _out_size(w, k, stride, pads[2], pads[3])
  y = torch.empty((n, c, oh, ow), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
  arg = torch.empty((n, oh, ow, c), dtype=torch.uint8, device=x.device)
  _check(_fn("agb_maxpool_forward", x)(_ptr(x), _ptr(y), _ptr(arg), ctypes.c_int(n), ctypes.c_int(h), ctypes.c_int(w), ctypes.c_int(c), ctypes.c_int(oh), ctypes.c_int(ow),
                                    ctypes.c_int(k), ctypes.c_int(stride), ctypes.c_int(pads[0]), ctypes.c_int(pads[2]), _stream()), "maxpool_forward")
  return y, arg


def maxpool_backward(dy, shape, arg, k, stride, pads):
  n, c, h, w = shape
  if not dy.is_contiguous(memory_format=torch.channels_last):
    dy = dy.contiguous(memory_format=torch.channels_last)
  oh, ow = dy.shape[2], dy.shape[3]
  dx = torch.empty((n, c, h, w), dtype=dy.dtype, device=dy.device, memory_format=torch.channels_last)
  _check(_fn("agb_maxpool_backward", dy)(_ptr(dy), _ptr(arg), _ptr(dx), ctypes.c_int(n), ctypes.c_int(h), ctypes.c_int(w), ctypes.c_int(c), ctypes.c_int(oh), ctypes.c_int(ow),
                                     ctypes.c_int(k), ctypes.c_int(stride), ctypes.c_int(pads[0]), ctypes.c_int(pads[2]), _stream()), "maxpool_backward")
  return dx


def global_avgpool_forward(x):
  if not enabled("pool") or not _cl_ok(x) or x.shape[1] % 8:
    return None
  n, c, h, w = x.shape
  y = torch.empty((n, c, 1, 1), dtype=x.dtype, device=x.device, memory_format=torch.channels_last)
  _check(_fn("agb_avgpool_forward", x)(_ptr(x), _ptr(y), ctypes.c_int(n), ctypes.c_int(h * w), ctypes.c_int(c), _stream()), "avgpool_forward")
  return y


def global_avgpool_backward(dy, shape):
  n, c, h, w = shape
  if not enabled("pool") or dy.dtype not in _DTYPES or c % 8:
    return None
  dy = dy.reshape(n, c).contiguous()
  dx = torch.empty((n, c, h, w), dtype=dy.dtype, device=dy.device, memory_format=torch.channels_last)
  _check(_fn("agb_avgpool_backward", dy)(_ptr(dy), _ptr(dx), ctypes.c_int(n), ctypes.c_int(h * w), ctypes.c_int(c), _stream()), "avgpool_backward")
  return dx


def softmax_xent(logits, labels, label_smoothing, groups=1):
  if not enabled("xent") or logits.dtype not in _DTYPES or logits.stride(1) != 1:
    return None
  batch, classes = logits.shape
  dlogits = torch.empty_strided(logits.shape, logits.stride(), dtype=logits.dtype, device=logits.device)
  loss = torch.empty((groups,) if groups > 1 else (), dtype=torch.float32, device=logits.device)
  labels = labels if labels.dtype == torch.int64 else labels.long()
  _check(_fn("agb_softmax_xent", logits)(_ptr(logits), _ptr(labels), _ptr(dlogits), _ptr(loss), ctypes.c_int(batch), ctypes.c_int(classes), ctypes.c_longlong(logits.stride(0)),
                                 ctypes.c_float(label_smoothing), ctypes.c_int(groups), _stream()), "softmax_xent")
  return loss, dlogits


_MEANS = {"vgg": (123.68, 116.78, 103.94, 1.0), "inception": (127.5, 127.5, 127.5, 1.0 / 127.5), "lenet": (128.0, 128.0, 128.0, 1.0 / 128.0)}


def image_normalize(images, mode, dtype):
  """uint8 NHWC -> bf16 channels_last (N, Cpad, H, W) with the channel dimension zero-padded to 8 (TMA/im2col friendly)."""
  if not enabled("image") or images.dtype != torch.uint8 or dtype not in _DTYPES or images.dim() != 4 or not images.is_contiguous():
    return None
  n, h, w, c = images.shape
  if c > 3:
    return None
  m0, m1, m2, scale = _MEANS.get(mode, _MEANS["lenet"])
  if mode == "vgg" and c != 3:
    m0, m1, m2, scale = _MEANS["lenet"]
  out = torch.empty((n, h, w, c), dtype=dtype, device=images.device)
  _check(_fn("agb_image_normalize", out)(_ptr(images), _ptr(out), ctypes.c_longlong(n * h * w), ctypes.c_int(c), ctypes.c_int(c), ctypes.c_float(m0), ctypes.c_float(m1),
                                    ctypes.c_float(m2), ctypes.c_float(scale), _stream()), "image_normalize")
  return out.permute(0, 3, 1, 2)

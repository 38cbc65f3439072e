"""Hopper GEMM and convolution kernels (native/op_nn/gemm_kernels.cuh, conv.cu) compared bit for bit with a float64 oracle.

Exactness argument. GEMM and convolution are sums of products. The operands below are small integers, or dyadic rationals
m * 2^-10 with |m| <= 2047 paired with a sparse +-1 operand. Every product is then an integer multiple of a known grid g
(1 for integers, 2^-10 for the dyadic cases, 2^-2 for the TF32 truncation probe), and so is every partial sum, in whatever order the
kernel adds them: k-blocks, mma fragments, split-K atomics, grouped chunks. A multiple of g is exact in fp32 while it stays
below 2^24 g, and every case asserts, before comparing, that the float64 reference stays below 2^12 g (`_on_grid`). That margin
also keeps the result exact if the tensor core aligns its internal sums to fewer than 24 bits. The float64 result is then the one
correct answer: fp32 outputs must equal it, bf16 outputs must equal its round-to-nearest-even bf16 value, with zero tolerance.
A wrong tile coordinate, a dropped or doubled k-block, a swizzle slip, a padding off-by-one, a parity mistake or a group offset
changes at least one element.
"""

import contextlib
import ctypes

import pytest
import torch
import torch.nn.functional as F

gpu = pytest.mark.gpu
CL = torch.channels_last
BF16, FP32 = torch.bfloat16, torch.float32
SENTINEL = -777.0          # fills the bytes around an output: a kernel must never write there
EXACT_UNITS = 2 ** 12      # largest |reference| in grid units that a case may have (see the module docstring)


# ---------------------------------------------------------------------------- #
# Seeded operand generators (drawn on the CPU, so that the same seed gives the same operands everywhere)

def _gen(seed):
  return torch.Generator().manual_seed(seed)


def _ints(shape, seed, dtype, device="cuda", lo=-4, hi=4):
  """Integers uniform in [lo, hi]: exact in bf16 and TF32, products exact and small."""
  return torch.randint(lo, hi + 1, tuple(shape), generator=_gen(seed)).to(dtype).to(device)


def _ternary(shape, seed, dtype, device="cuda"):
  """{-1, 0, 1}: for long sums, whose partial sums would outgrow the exact range with wider integers."""
  return _ints(shape, seed, dtype, device, -1, 1)


def _operand(shape, seed, dtype, depth, device="cuda"):
  """Integer operand for sums of up to `depth` products: [-4, 4] while that keeps the sums far inside the exact range, else ternary."""
  return (_ints if depth <= 1024 else _ternary)(shape, seed, dtype, device)


def _dyadic(shape, seed, device="cuda"):
  """m * 2^-10 with |m| <= 2047: exact in TF32 (11-bit significand), mostly not exact in bf16 (8 bits)."""
  return (torch.randint(-2047, 2048, tuple(shape), generator=_gen(seed)).double() * 2.0 ** -10).float().to(device)


def _sparse_signs(shape, seed, dim, dtype, device="cuda", per_line=2):
  """+-1 at `per_line` random positions along dimension `dim` of every line, zero elsewhere: each output of a product with it sums
  at most `per_line` terms."""
  gen = _gen(seed)
  moved = list(shape)
  moved[dim], moved[-1] = moved[-1], moved[dim]
  lines = 1
  for s in moved[:-1]:
    lines *= s
  length = moved[-1]
  t = torch.zeros((lines, length), dtype=torch.float64)
  for _ in range(per_line):
    pos = torch.randint(0, length, (lines,), generator=gen)
    sign = torch.randint(0, 2, (lines,), generator=gen).double() * 2 - 1
    t[torch.arange(lines), pos] = sign
  return t.view(moved).transpose(dim, -1).contiguous().to(dtype).to(device)


# ---------------------------------------------------------------------------- #
# Oracle and comparison

def _on_grid(ref, grid=1.0):
  """The float64 reference snapped to its grid (keeps fp64 library rounding out of the oracle), with the exactness precondition."""
  units = ref / grid
  snapped = torch.round(units)
  moved = float((snapped - units).abs().max()) if units.numel() else 0.0
  assert moved <= 1e-9, "float64 reference is off its grid by %g units" % moved
  largest = float(snapped.abs().max()) if units.numel() else 0.0
  assert largest < EXACT_UNITS, "operands too dense for an exact comparison: max |reference| = %g grid units" % largest
  return snapped * grid


def _assert_exact(out, ref, what="", bn=128):
  """`out` (fp32 or bf16, 2-D) must equal the float64 `ref` converted to its dtype, bit for bit. On failure: the first bad (row, col),
  its tile (row // 128, col // bn) and the set of bad tiles."""
  assert out.dim() == 2 and out.shape == ref.shape, (what, tuple(out.shape), tuple(ref.shape))
  want = ref.to(out.dtype)
  if torch.equal(out, want):
    return
  bad = (out != want) & ~(torch.isnan(out) & torch.isnan(want))
  where = bad.nonzero()
  r, c = int(where[0, 0]), int(where[0, 1])
  tiles = sorted({(i // 128, j // bn) for i, j in where[:4096].tolist()})
  raise AssertionError("%s: %d of %d elements differ; first at (row %d, col %d) = tile (%d, %d): got %r, want %r; bad tiles %s%s"
                       % (what, int(bad.sum()), out.numel(), r, c, r // 128, c // bn, float(out[r, c]), float(want[r, c]), tiles[:16],
                          " ..." if len(tiles) > 16 else ""))


def _nhwc_rows(t):
  """(N, C, H, W) activation -> [N*H*W, C] rows (the GEMM view the kernels tile)."""
  return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


def _gemm_ref(layout, a, b):
  a, b = a.double(), b.double()
  return {"nt": lambda: a @ b.t(), "nn": lambda: a @ b, "tn": lambda: a.t() @ b}[layout]()


def _gemm_shapes(layout, m, n, k):
  return {"nt": ((m, k), (n, k)), "nn": ((m, k), (k, n)), "tn": ((k, m), (k, n))}[layout]


# ---------------------------------------------------------------------------- #
# Convolution reference without cuDNN: patch rows in (kh, kw, c) column order, as `nn_native._weight_rows` lays out the weights

def _out_size(size, k, stride, lo, hi):
  return (size + lo + hi - k) // stride + 1


def _patch_rows(x, kh, kw, stride, pads):
  """[N*OH*OW, kh*kw*C] patches of x (N, C, H, W); pads = (top, bottom, left, right)."""
  t, b, l, r = pads
  n, c = x.shape[:2]
  cols = F.unfold(F.pad(x, (l, r, t, b)), (kh, kw), stride=stride)   # [N, C*kh*kw, L], columns (c, kh, kw)
  return cols.view(n, c, kh, kw, -1).permute(0, 4, 2, 3, 1).reshape(-1, kh * kw * c)


def conv_forward_ref(x, w, stride, pads):
  """x (N, Cin, H, W), w [Cout, kh, kw, Cin] -> y (N, Cout, OH, OW), all float64."""
  n, _, h, wd = x.shape
  cout, kh, kw, _ = w.shape
  oh, ow = _out_size(h, kh, stride, pads[0], pads[1]), _out_size(wd, kw, stride, pads[2], pads[3])
  y = _patch_rows(x, kh, kw, stride, pads) @ w.reshape(cout, -1).t()
  return y.view(n, oh, ow, cout).permute(0, 3, 1, 2)


def conv_wgrad_ref(dy, x, kh, kw, stride, pads, groups=1):
  """[groups, Cout, kh, kw, Cin]: dy^T @ patches(x) over each group's consecutive images."""
  cout, cin = dy.shape[1], x.shape[1]
  cols = _patch_rows(x, kh, kw, stride, pads).view(groups, -1, kh * kw * cin)
  rows = _nhwc_rows(dy).view(groups, -1, cout)
  return (rows.transpose(1, 2) @ cols).view(groups, cout, kh, kw, cin)


def conv_dgrad_ref(dy, w, x_shape, stride, pads):
  """fold(dy @ W) with the padding cropped: dx (N, Cin, H, W)."""
  n, c, h, wd = x_shape
  cout, kh, kw, _ = w.shape
  t, b, l, r = pads
  dcols = _nhwc_rows(dy) @ w.reshape(cout, -1)                                 # [N*L, kh*kw*Cin], columns (kh, kw, c)
  dcols = dcols.view(n, -1, kh, kw, c).permute(0, 4, 2, 3, 1).reshape(n, c * kh * kw, -1)
  dxp = F.fold(dcols, (h + t + b, wd + l + r), (kh, kw), stride=stride)
  return dxp[:, :, t:t + h, l:l + wd]


@pytest.mark.parametrize("stride,pads,kh,kw", [(1, (1, 1, 1, 1), 3, 3), (2, (1, 1, 1, 1), 3, 3), (1, (0, 1, 0, 1), 3, 3), (2, (0, 1, 0, 1), 3, 3),
                                               (1, (1, 1, 0, 0), 3, 1), (2, (1, 2, 0, 1), 3, 2), (2, (3, 3, 3, 3), 7, 7)])
def test_conv_oracle_matches_conv2d(stride, pads, kh, kw):
  """The unfold / fold reference against `F.conv2d` and its autograd in float64 (integer data: both sides are exact)."""
  n, cin, cout, h, wd = 2, 5, 6, 9, 8
  x = _ints((n, cin, h, wd), 1, torch.float64, "cpu")
  w = _ints((cout, kh, kw, cin), 2, torch.float64, "cpu")
  t, b, l, r = pads
  xp = F.pad(x, (l, r, t, b)).requires_grad_(True)
  wt = w.permute(0, 3, 1, 2).clone().requires_grad_(True)
  y = F.conv2d(xp, wt, stride=stride)
  assert torch.equal(conv_forward_ref(x, w, stride, pads), y.detach())
  dy = _ints(tuple(y.shape), 3, torch.float64, "cpu")
  y.backward(dy)
  assert torch.equal(conv_wgrad_ref(dy, x, kh, kw, stride, pads)[0], wt.grad.permute(0, 2, 3, 1))
  assert torch.equal(conv_dgrad_ref(dy, w, x.shape, stride, pads), xp.grad[:, :, t:t + h, l:l + wd])
  # per-group weight gradients are the gradients of each group's images alone
  grouped = conv_wgrad_ref(dy, x, kh, kw, stride, pads, groups=2)
  assert torch.equal(grouped.sum(dim=0), wt.grad.permute(0, 2, 3, 1))
  assert torch.equal(grouped[1], conv_wgrad_ref(dy[1:], x[1:], kh, kw, stride, pads)[0])


def test_grid_precondition_rejects_dense_operands():
  """The oracle refuses references it cannot vouch for: off-grid values and magnitudes beyond the exact range."""
  _on_grid(torch.tensor([[4095.0, -3.0]], dtype=torch.float64))
  with pytest.raises(AssertionError):
    _on_grid(torch.tensor([[4096.0]], dtype=torch.float64))
  with pytest.raises(AssertionError):
    _on_grid(torch.tensor([[0.5]], dtype=torch.float64))
  with pytest.raises(AssertionError):
    _assert_exact(torch.tensor([[1.0, 2.0]]), torch.tensor([[1.0, 3.0]], dtype=torch.float64), "probe")


# ---------------------------------------------------------------------------- #
# Argument validation of the grouped weight-gradient GEMM (host side: runs without a GPU)

def test_mm_tn_rejects_rows_not_divisible_by_groups():
  from aggregathor_b200.ops import nn_native as nat
  x, y = torch.zeros((10, 8), dtype=BF16), torch.zeros((10, 16), dtype=BF16)
  out = torch.zeros((3, 8 * 16))
  with pytest.raises(ValueError, match="groups"):
    nat.mm_tn(x, y, out=out[0].view(8, 16), groups=3, group_stride=out.stride(0))


def test_mm_tn_rejects_groups_sharing_one_output():
  from aggregathor_b200.ops import nn_native as nat
  x, y = torch.zeros((12, 8), dtype=BF16), torch.zeros((12, 16), dtype=BF16)
  out = torch.zeros((3, 8 * 16))
  with pytest.raises(ValueError, match="group_stride"):
    nat.mm_tn(x, y, groups=3)
  with pytest.raises(ValueError, match="group_stride"):
    nat.mm_tn(x, y, out=out[0].view(8, 16), groups=3, group_stride=0)
  with pytest.raises(ValueError, match="group_stride"):
    nat.mm_tn(x, y, out=out[0].view(8, 16), groups=3, group_stride=8 * 16 - 1)   # overlapping outputs


# ---------------------------------------------------------------------------- #
# GEMM matrix

@contextlib.contextmanager
def _gemm_mode(persistent=True, wide=True):
  from aggregathor_b200.ops import nn_native as nat
  nat.set_gemm_persistent(persistent)
  nat._lib().agb_gemm_set_wide_tiles(ctypes.c_int(1 if wide else 0))
  try:
    yield
  finally:
    nat.set_gemm_persistent(True)
    nat._lib().agb_gemm_set_wide_tiles(ctypes.c_int(1))


# (bn, wide tiles): the automatic choice with 128 x 256 tiles allowed and disallowed, then every forced width (TF32 maps 256 to 128)
BN_VARIANTS = [(0, True), (0, False), (64, True), (128, True), (256, True)]


def _kblocks(k, dtype):
  return -(-k // (64 if dtype == BF16 else 32))


# M, N in {1, 7, 127, 128, 129, 257, 1000} (odd N included), K in {8, 56, 64, 72, 1000, 4096}: tails of every dimension in every
# layout, MN-major M and N below one 64-element chunk, and one shape large enough for the automatic 128 x 256 tiles.
GEMM_SHAPES = [(1, 1, 8), (7, 1000, 56), (127, 129, 64), (128, 128, 72), (129, 257, 1000), (257, 7, 4096), (1000, 127, 72), (128, 1, 1000),
               (1, 128, 4096), (257, 129, 8), (1000, 1000, 64), (3072, 1000, 72)]


@gpu
@pytest.mark.parametrize("dtype", [BF16, FP32], ids=["bf16", "tf32"])
@pytest.mark.parametrize("layout", ["nt", "nn", "tn"])
@pytest.mark.parametrize("m,n,k", GEMM_SHAPES)
def test_gemm_exact(layout, dtype, m, n, k):
  """Every layout x tile width x wide tiles on / off x persistent / tile-per-CTA launch (x split-K for TN) is bit-exact."""
  from aggregathor_b200.ops import nn_native as nat
  sa, sb = _gemm_shapes(layout, m, n, k)
  a, b = _operand(sa, 11 + m, dtype, k), _operand(sb, 12 + n, dtype, k)
  ref = _on_grid(_gemm_ref(layout, a, b))
  splits_list = [1, 2, 3, None, _kblocks(k, dtype) + 3] if layout == "tn" else [1]
  for persistent in (True, False):
    for bn, wide in BN_VARIANTS:
      with _gemm_mode(persistent, wide):
        for splits in splits_list:
          what = "%s %s persistent=%d bn=%d wide=%d splits=%s" % (layout, dtype, persistent, bn, wide, splits)
          tile_n = min(bn or 128, 128 if dtype == FP32 else 256)
          if layout == "tn":
            _assert_exact(nat.mm_tn(a, b, splits=splits, bn=bn), ref, what, tile_n)
          elif layout == "nt":
            _assert_exact(nat.mm_nt(a, b, bn=bn, out_dtype=FP32), ref, what, tile_n)
          else:
            _assert_exact(nat.mm_nn(a, b, bn=bn, out_dtype=FP32), ref, what, tile_n)
          if dtype == BF16 and layout != "tn":
            out = (nat.mm_nt if layout == "nt" else nat.mm_nn)(a, b, bn=bn)
            assert out.dtype == BF16
            _assert_exact(out, ref, what + " bf16 out", tile_n)


@gpu
@pytest.mark.parametrize("dtype", [BF16, FP32], ids=["bf16", "tf32"])
def test_split_k_edges(dtype):
  """More splits than K blocks (clamped), and a split count whose ceil-divided ranges would leave the last split empty."""
  from aggregathor_b200.ops import nn_native as nat
  kb = 64 if dtype == BF16 else 32
  for m, n, k, splits in ((129, 200, 5 * kb, 4), (129, 200, 5 * kb, 5), (64, 72, 3 * kb - 5, 7), (300, 7, kb, 9), (33, 257, 7 * kb + 1, 6)):
    a, b = _ints((k, m), m + k, dtype), _ints((k, n), n + k, dtype)
    ref = _on_grid(_gemm_ref("tn", a, b))
    for persistent in (True, False):
      with _gemm_mode(persistent):
        _assert_exact(nat.mm_tn(a, b, splits=splits), ref, "m=%d n=%d k=%d splits=%d persistent=%d" % (m, n, k, splits, persistent))


@gpu
@pytest.mark.parametrize("dtype", [BF16, FP32], ids=["bf16", "tf32"])
@pytest.mark.parametrize("groups", [1, 3, 8])
@pytest.mark.parametrize("m,n,kg", [(96, 160, 100), (257, 129, 40), (7, 64, 1000), (130, 256, 392)])
def test_grouped_mm_tn_exact(dtype, groups, m, n, kg):
  """Grouped weight gradients: each group's K range (not a multiple of the K block) ends exactly where the 3-D tensor map
  zero-fills; no group's rows leak into its neighbour's output; nothing is written between the groups' outputs."""
  from aggregathor_b200.ops import nn_native as nat
  a, b = _operand((groups * kg, m), 21 + m, dtype, kg), _operand((groups * kg, n), 22 + n, dtype, kg)
  refs = [_on_grid(_gemm_ref("tn", a[g * kg:(g + 1) * kg], b[g * kg:(g + 1) * kg])) for g in range(groups)]
  for pad in (8, 3):   # even group stride (paired stores when N is even) and odd group stride (scalar epilogue)
    stride = m * n + pad
    buf = torch.empty(groups * stride + 16, device="cuda")
    out = buf[:m * n].view(m, n)
    for splits in (1, None, 3):
      for bn in (0, 64):
        buf.fill_(SENTINEL)
        nat.mm_tn(a, b, out=out, splits=splits, bn=bn, groups=groups, group_stride=stride)
        for g in range(groups):
          _assert_exact(buf[g * stride:g * stride + m * n].view(m, n), refs[g], "group %d/%d stride %d splits %s bn %d" % (g, groups, stride, splits, bn))
          assert bool((buf[g * stride + m * n:(g + 1) * stride] == SENTINEL).all()), ("write between groups", g, stride, splits)
        assert bool((buf[groups * stride:] == SENTINEL).all()), "write past the last group"


@gpu
@pytest.mark.parametrize("dtype", [BF16, FP32], ids=["bf16", "tf32"])
@pytest.mark.parametrize("m,n,k", [(129, 257, 72), (7, 1, 1000), (1000, 127, 64), (3072, 1000, 72)])
def test_bias_relu_epilogue(dtype, m, n, k):
  """fp32 bias + ReLU with fp32 output, and bias with bf16 output (bf16 only), for every tile width."""
  from aggregathor_b200.ops import nn_native as nat
  x, w = _operand((m, k), 31, dtype, k), _operand((n, k), 32, dtype, k)
  bias = _ints((n,), 33, FP32, lo=-8, hi=8)
  acc = _gemm_ref("nt", x, w) + bias.double()
  relu_ref, bias_ref = _on_grid(torch.relu(acc)), _on_grid(acc)
  for bn, wide in BN_VARIANTS:
    with _gemm_mode(True, wide):
      _assert_exact(nat.mm_nt(x, w, bias=bias, relu=True, bn=bn, out_dtype=FP32), relu_ref, "bias+relu bn=%d wide=%d" % (bn, wide))
      _assert_exact(nat.mm_nt(x, w, bias=bias, bn=bn, out_dtype=FP32), bias_ref, "bias bn=%d wide=%d" % (bn, wide))
      if dtype == BF16:
        _assert_exact(nat.mm_nt(x, w, bias=bias, bn=bn), bias_ref, "bias bf16 out bn=%d wide=%d" % (bn, wide))
        _assert_exact(nat.mm_nt(x, w, bias=bias, relu=True, bn=bn), relu_ref, "bias+relu bf16 out bn=%d wide=%d" % (bn, wide))


@gpu
@pytest.mark.parametrize("layout", ["nt", "nn"])
def test_bf16_output_rounds_ties_to_even(layout):
  """Exact results that are odd integers in [257, 511] (and their negatives) sit halfway between two bf16 values (spacing 2): the
  epilogue must round them to even, as `Tensor.to(torch.bfloat16)` does, on the paired and on the scalar store path."""
  from aggregathor_b200.ops import nn_native as nat
  m, n, k = 300, 200, 72
  sa, sb = _gemm_shapes(layout, m, n, k)
  a, b = _ints(sa, 41, BF16, lo=-2, hi=2), _ints(sb, 42, BF16, lo=-2, hi=2)
  # one k column of ones in A times an offset of +-384 in B moves every result into [257, 511] or its negative
  offset = torch.where(torch.arange(n, device="cuda") % 3 == 0, -384.0, 384.0).to(BF16)
  a[:, 0] = 1
  if layout == "nt":
    b[:, 0] = offset
  else:
    b[0, :] = offset
  ref = _on_grid(_gemm_ref(layout, a, b))
  odd = ref.abs().remainder(2) == 1
  assert int(odd.sum()) > m * n // 4 and float(ref.abs().min()) > 256 and float(ref.abs().max()) < 512
  mm = nat.mm_nt if layout == "nt" else nat.mm_nn
  for bn in (64, 128, 256):
    _assert_exact(mm(a, b, bn=bn), ref, "ties bn=%d" % bn)
    buf = torch.full((m * (n + 1) + 2,), SENTINEL, dtype=BF16, device="cuda")
    out = buf[1:].as_strided((m, n), (n + 1, 1))      # odd ldc, 2 bytes off: scalar stores
    mm(a, b, out=out, bn=bn)
    _assert_exact(out, ref, "ties scalar bn=%d" % bn)


@gpu
@pytest.mark.parametrize("dtype", [BF16, FP32], ids=["bf16", "tf32"])
def test_output_addressing(dtype):
  """Padded output rows, odd ldc, a C that starts 4 bytes (fp32) or 2 bytes (bf16) into its allocation: the latter two turn the paired
  epilogue off (scalar stores, scalar split-K atomics). Bias must still be applied, and nothing outside C may change."""
  from aggregathor_b200.ops import nn_native as nat
  m, n, k = 257, 130, 200
  x, w = _ints((m, k), 51, dtype), _ints((n, k), 52, dtype)
  bias = _ints((n,), 53, FP32, lo=-8, hi=8)
  ref = _on_grid(_gemm_ref("nt", x, w) + bias.double())
  out_types = (FP32, BF16) if dtype == BF16 else (FP32,)
  for out_dtype in out_types:
    padded = nat.alloc_out(m, n - 1, out_dtype, "cuda")
    assert padded.stride(0) % 8 == 0 and padded.stride(0) > n - 1
    nat.mm_nt(x, w[:n - 1], bias=bias[:n - 1], out=padded)
    _assert_exact(padded, ref[:, :n - 1], "alloc_out %s" % out_dtype)
    for ldc, offset in ((n + 1, 0), (n, 1), (n + 3, 1)):
      buf = torch.full((m * ldc + offset + 8,), SENTINEL, dtype=out_dtype, device="cuda")
      out = buf[offset:].as_strided((m, n), (ldc, 1))
      for bn in (64, 128, 256):
        buf.fill_(SENTINEL)
        nat.mm_nt(x, w, bias=bias, out=out, bn=bn)
        what = "%s ldc=%d offset=%d bn=%d" % (out_dtype, ldc, offset, bn)
        _assert_exact(out, ref, what)
        written = torch.zeros_like(buf, dtype=torch.bool)
        written[offset:].as_strided((m, n), (ldc, 1)).fill_(True)
        assert bool((buf[~written] == SENTINEL).all()), "write outside C: " + what
  # split-K weight gradient into a misaligned C: scalar fp32 atomics
  a, b = _ints((1000, 129), 54, dtype), _ints((1000, 64), 55, dtype)
  ref = _on_grid(_gemm_ref("tn", a, b))
  for ldc, offset in ((64, 1), (65, 0)):
    buf = torch.full((129 * ldc + offset + 8,), SENTINEL, device="cuda")
    out = buf[offset:].as_strided((129, 64), (ldc, 1))
    for splits in (1, 3, None):
      nat.mm_tn(a, b, out=out, splits=splits)
      _assert_exact(out, ref, "tn ldc=%d offset=%d splits=%s" % (ldc, offset, splits))


@gpu
@pytest.mark.parametrize("dtype", [BF16, FP32], ids=["bf16", "tf32"])
def test_strided_operands(dtype):
  """Operands that `_rows` must copy (row stride not a multiple of 8, misaligned base, transposed view) give the exact product."""
  from aggregathor_b200.ops import nn_native as nat
  m, n, k = 200, 96, 150
  big = _ints((m + 1, k + 11), 61, dtype)
  wide_w = _ints((n, k + 5), 62, dtype)
  for x in (big[:m, :k], big[1:, 1:k + 1], _ints((k, m), 63, dtype).t()):
    w = wide_w[:, :k]
    _assert_exact(nat.mm_nt(x, w, out_dtype=FP32), _on_grid(_gemm_ref("nt", x, w)), "nt %s" % (x.stride(),))
    _assert_exact(nat.mm_nn(x, w.t(), out_dtype=FP32), _on_grid(_gemm_ref("nn", x, w.t())), "nn %s" % (x.stride(),))
    _assert_exact(nat.mm_tn(x.t(), w.t()), _on_grid(_gemm_ref("tn", x.t(), w.t())), "tn %s" % (x.stride(),))


@gpu
@pytest.mark.parametrize("dtype", [BF16, FP32], ids=["bf16", "tf32"])
@pytest.mark.parametrize("layout", ["nt", "nn", "tn", "nt+relu"])
def test_nonfinite_inputs_stay_in_their_row_and_column(layout, dtype):
  """Inf in one row of A and NaN in one column of B: exactly the outputs in that row or column are non-finite, and every other
  output is still exact. Catches contamination across tiles, k-splits or work items through the reused shared-memory ring.
  `nt+relu`: the epilogue ReLU keeps NaN and +inf and maps -inf to 0, so in the inf row only the outputs whose B entry is
  positive (+inf) or zero (inf * 0 = NaN) stay non-finite."""
  from aggregathor_b200.ops import nn_native as nat
  relu = layout == "nt+relu"
  layout = "nt" if relu else layout
  m, n, k = 300, 260, 1000
  row, col, k_inf, k_nan = 131, 70, 5, 900
  sa, sb = _gemm_shapes(layout, m, n, k)
  a, b = _ints(sa, 71, dtype), _ints(sb, 72, dtype)
  ref = _gemm_ref(layout, a, b)
  if layout == "tn":
    a[k_inf, row] = float("inf")
  else:
    a[row, k_inf] = float("inf")
  if layout == "nt":
    b[col, k_nan] = float("nan")
  else:
    b[k_nan, col] = float("nan")
  expect = torch.zeros((m, n), dtype=torch.bool, device="cuda")
  expect[row, :] = True
  expect[:, col] = True
  ref = _on_grid(ref.masked_fill(expect, 0))
  nonfinite = expect
  if relu:
    ref = torch.relu(ref)
    inf_row = float("inf") * b[:, k_inf].double()   # the inf term of each output of the row; the finite terms cannot change it
    nonfinite = expect.clone()
    nonfinite[row, :] = torch.isnan(inf_row) | (inf_row > 0)
    nonfinite[:, col] = True
  for persistent in (True, False):
    for bn, wide in BN_VARIANTS:
      with _gemm_mode(persistent, wide):
        for splits in ((1, 4, None) if layout == "tn" else (1,)):
          what = "%s persistent=%d bn=%d splits=%s" % (layout, persistent, bn, splits)
          if layout == "tn":
            out = nat.mm_tn(a, b, splits=splits, bn=bn)
          else:
            out = nat.mm_nt(a, b, relu=relu, bn=bn, out_dtype=FP32) if layout == "nt" else nat.mm_nn(a, b, bn=bn, out_dtype=FP32)
          bad = ~torch.isfinite(out)
          assert torch.equal(bad, nonfinite), (what, int((bad != nonfinite).sum()), (bad != nonfinite).nonzero()[:8].tolist())
          _assert_exact(out.masked_fill(expect, 0), ref, what)


@gpu
@pytest.mark.parametrize("dtype", [BF16, FP32], ids=["bf16", "tf32"])
def test_dependent_gemm_chain_under_pdl(dtype):
  """Programmatic dependent launch: forward, data-gradient and weight-gradient GEMMs, each reading the previous output, issued back
  to back. Every kernel that starts early must wait for its producer; the final result is exact."""
  from aggregathor_b200.ops import nn_native as nat
  m, k, n1, n2, n3 = 512, 320, 384, 200, 136
  x = _ints((m, k), 81, dtype)
  w1 = _sparse_signs((n1, k), 82, 1, dtype)       # each output of the first GEMM sums 2 terms: |h1| <= 8
  w2 = _sparse_signs((n1, n2), 83, 0, dtype)      # |h2| <= 16
  z = _ternary((m, n3), 84, dtype)
  h1 = _gemm_ref("nt", x, w1).to(dtype).double()
  h2 = _gemm_ref("nn", h1, w2).to(dtype).double()
  ref = _on_grid(_gemm_ref("tn", h2, z))
  nat.set_launch_overlap(True)
  try:
    outs = []
    for _ in range(3):
      g1 = nat.mm_nt(x, w1)
      g2 = nat.mm_nn(g1, w2)
      outs.append(nat.mm_tn(g2, z))
    torch.cuda.synchronize()
  finally:
    nat.set_launch_overlap(False)
  for i, out in enumerate(outs):
    _assert_exact(out, ref, "chain %d" % i)


# ---------------------------------------------------------------------------- #
# Convolutions through `ops.nn` with backend "native": the dispatch that training uses

def _conv_case(dtype, n, cin, cout, kh, kw, h, w, stride, pads, path, groups=1, has_bias=True, need_dx=True, seed=0, split_modes=(False,)):
  """Forward (bias + ReLU), weight gradient (per group), bias gradient and data gradient of one convolution, each bit-exact.
  `path`: "implicit", "im2col" or "pointwise", the native route this case must take."""
  from aggregathor_b200.ops import nn as ops
  from aggregathor_b200.ops import nn_native as nat
  oh, ow = _out_size(h, kh, stride, pads[0], pads[1]), _out_size(w, kw, stride, pads[2], pads[3])
  depth = max(kh * kw * max(cin, cout), n // groups * oh * ow)
  x = _operand((n, cin, h, w), seed + 1, dtype, depth).contiguous(memory_format=CL)
  wt = _operand((cout, kh, kw, cin), seed + 2, dtype, depth).contiguous()
  bias = _ints((cout,), seed + 3, FP32, lo=-8, hi=8)
  dy = _operand((n, cout, oh, ow), seed + 4, dtype, depth).contiguous(memory_format=CL)
  taken = "pointwise" if nat._is_pointwise(wt, stride, pads) else "implicit" if nat._implicit_ok(x, wt, stride, pads) else "im2col"
  assert taken == path, (taken, path)
  what = "%s n=%d %dx%dx%d -> %d k=%dx%d s=%d pads=%s groups=%d" % (dtype, n, h, w, cin, cout, kh, kw, stride, pads, groups)

  x64, w64 = x.double(), wt.double()
  y_ref = _on_grid(torch.relu(conv_forward_ref(x64, w64, stride, pads) + bias.double().view(1, -1, 1, 1)))
  before = dict(ops.fallbacks)
  y = ops.conv2d_forward("native", x, wt, bias, stride, pads, True)
  assert y.dtype == dtype
  _assert_exact(_nhwc_rows(y), _nhwc_rows(y_ref), "forward " + what)

  dym = dy.double() * (y > 0).double()   # the ReLU mask of the native output, as `test_conv` takes it (equal to the oracle's here)
  gw_ref = _on_grid(conv_wgrad_ref(dym, x64, kh, kw, stride, pads, groups))
  gb_ref = _on_grid(_nhwc_rows(dym).view(groups, -1, cout).sum(dim=1))
  dx_ref = _on_grid(conv_dgrad_ref(dym, w64, x.shape, stride, pads)) if need_dx else None
  numel = cout * kh * kw * cin
  stride_g = numel + cout + 8      # one worker's row of the gradient matrix
  rows = torch.empty((groups, stride_g), device="cuda")
  for deterministic in split_modes:
    nat.set_deterministic(deterministic)
    try:
      rows.fill_(SENTINEL)
      gw, gb = rows[0, :numel].view(cout, kh, kw, cin), rows[0, numel:numel + cout]
      dx, _, _ = ops.conv2d_backward("native", dy, x, wt, y, stride, pads, True, has_bias, need_dx, gw, gb, groups, stride_g)
    finally:
      nat.set_deterministic(False)
    tag = "%s deterministic=%d" % (what, deterministic)
    for g in range(groups):
      _assert_exact(rows[g, :numel].view(cout, -1), gw_ref[g].reshape(cout, -1), "wgrad group %d %s" % (g, tag))
      if has_bias:
        _assert_exact(rows[g, numel:numel + cout].view(1, -1), gb_ref[g].view(1, -1), "bias grad group %d %s" % (g, tag))
    assert bool((rows[:, numel + (cout if has_bias else 0):] == SENTINEL).all()), "write past a worker's gradient " + tag
    if need_dx:
      assert dx.dtype == dtype and dx.shape == x.shape
      _assert_exact(_nhwc_rows(dx), _nhwc_rows(dx_ref), "dgrad " + tag)
  assert ops.fallbacks == before, "served by the aten provider: " + what


def _tf_same(k, stride=2):
  """TF "SAME" padding of an even map at stride 2: (top, bottom, left, right)."""
  total = max(k - stride, 0)
  return (total // 2, total - total // 2, total // 2, total - total // 2)


def _sym(k):
  p = (k - 1) // 2
  return (p, p, p, p)


# (cin, cout, k, stride, map, pads, n) for bf16; TF32 runs the same geometry with half the channels (multiples of 32)
IMPLICIT_CASES = [
  (64, 64, 3, 1, 56, _sym(3), 2), (64, 128, 5, 1, 28, _sym(5), 2), (128, 64, 7, 1, 14, _sym(7), 4), (64, 192, 3, 1, 7, _sym(3), 4),
  (192, 64, 3, 1, 5, _sym(3), 8), (64, 64, 5, 1, 3, _sym(5), 8), (128, 128, 7, 1, 7, _sym(7), 2), (64, 64, 3, 1, 3, _sym(3), 16),
  (64, 64, 2, 2, 56, _sym(2), 2), (64, 128, 3, 2, 28, _sym(3), 2), (128, 64, 3, 2, 14, (0, 1, 0, 1), 4), (64, 64, 4, 2, 28, _sym(4), 2),
  (64, 192, 5, 2, 14, _sym(5), 4), (192, 64, 5, 2, 28, _tf_same(5), 2), (64, 64, 3, 2, 56, (0, 1, 0, 1), 2), (128, 128, 2, 2, 14, _sym(2), 4),
  (64, 128, 4, 2, 14, (2, 1, 2, 1), 4), (64, 64, 3, 2, 6, _sym(3), 8)]


@gpu
@pytest.mark.parametrize("dtype", [BF16, FP32], ids=["bf16", "tf32"])
@pytest.mark.parametrize("cin,cout,k,stride,hw,pads,n", IMPLICIT_CASES)
def test_implicit_conv_exact(dtype, cin, cout, k, stride, hw, pads, n):
  """Implicit-GEMM convolution: 4-D TMA pixel boxes (smaller than the tile on 7, 5 and 3 maps), TMA element strides at stride 2,
  the parity-split data gradient, N tails (192 and, in TF32, 96 channels)."""
  scale = 1 if dtype == BF16 else 2
  _conv_case(dtype, n, cin // scale, cout // scale, k, k, hw, hw, stride, pads, "implicit", seed=cin + cout + k + hw, split_modes=(False, True))


# grouped weight gradients: (n images, cin, cout, k, stride, map, pads, groups)
GROUPED_CASES = [
  # ResNet-50 with 8 logical workers: per-worker batch 32 at 14x14x256 and 7x7x512, a reduced batch at 56x56x64, the stride-2 3x3
  # down-sampling layers, 1x1 pointwise layers (grouped mm_tn + grouped colsum) and the 7x7/2 stem at reduced resolution (im2col)
  (256, 256, 256, 3, 1, 14, _sym(3), 8), (256, 512, 512, 3, 1, 7, _sym(3), 8), (32, 64, 64, 3, 1, 56, _sym(3), 8),
  (32, 64, 64, 3, 2, 56, _sym(3), 8), (64, 128, 128, 3, 2, 28, _sym(3), 8), (256, 256, 256, 3, 2, 14, _sym(3), 8),
  (32, 256, 64, 1, 1, 56, (0, 0, 0, 0), 8), (256, 1024, 256, 1, 1, 14, (0, 0, 0, 0), 8), (16, 3, 64, 7, 2, 64, (3, 3, 3, 3), 8),
  (8, 64, 128, 3, 1, 28, _sym(3), 2), (8, 128, 64, 3, 2, 14, (0, 1, 0, 1), 2), (16, 64, 192, 5, 1, 7, _sym(5), 2)]


@gpu
@pytest.mark.parametrize("dtype", [BF16, FP32], ids=["bf16", "tf32"])
@pytest.mark.parametrize("n,cin,cout,k,stride,hw,pads,groups", GROUPED_CASES)
def test_grouped_conv_exact(dtype, n, cin, cout, k, stride, hw, pads, groups):
  """Per-worker weight gradients of a batched-workers step (one launch for all groups), with automatic split-K and with split-K off."""
  if dtype == FP32 and n * cin * hw * hw > 2 ** 23:
    n //= 4   # TF32 activations are twice as large: fewer images per worker
  path = "pointwise" if k == 1 else "im2col" if cin % (64 if dtype == BF16 else 32) else "implicit"
  _conv_case(dtype, n, cin, cout, k, k, hw, hw, stride, pads, path, groups=groups, need_dx=cin % 8 == 0, seed=n + cin + k, split_modes=(False, True))


@gpu
@pytest.mark.parametrize("dtype", [BF16, FP32], ids=["bf16", "tf32"])
@pytest.mark.parametrize("cin,cout,kh,kw,stride,h,w,pads", [
  (64, 96, 1, 7, 1, 17, 17, (0, 0, 3, 3)), (64, 96, 7, 1, 1, 17, 17, (3, 3, 0, 0)), (40, 64, 3, 1, 1, 12, 10, (1, 1, 0, 0)),
  (24, 48, 3, 3, 1, 14, 14, (1, 1, 1, 1)), (64, 64, 3, 3, 2, 15, 15, (0, 0, 0, 0)), (64, 128, 3, 3, 2, 7, 7, (1, 1, 1, 1)),
  (48, 64, 5, 5, 2, 13, 11, (2, 2, 2, 2))])
def test_im2col_conv_exact(dtype, cin, cout, kh, kw, stride, h, w, pads):
  """Convolutions the implicit kernels do not take (rectangular filters, Cin not a multiple of 64, stride 2 on odd maps): im2col +
  GEMM + col2im."""
  _conv_case(dtype, 4, cin, cout, kh, kw, h, w, stride, pads, "im2col", groups=2, seed=cin * kh + kw)


@gpu
@pytest.mark.parametrize("dtype", [BF16, FP32], ids=["bf16", "tf32"])
@pytest.mark.parametrize("groups", [1, 3])
def test_pointwise_conv_and_linear_exact(dtype, groups):
  """1x1 stride-1 convolutions and dense layers: mm_nt forward, grouped mm_tn + colsum weight and bias gradients, mm_nn data gradient."""
  from aggregathor_b200.ops import nn as ops
  _conv_case(dtype, 6, 136, 72, 1, 1, 9, 9, 1, (0, 0, 0, 0), "pointwise", groups=groups, seed=groups)
  batch, fin, fout = 30 * groups, 200, 72
  x, w = _ints((batch, fin), 91, dtype), _ints((fout, fin), 92, dtype)
  bias = _ints((fout,), 93, FP32, lo=-8, hi=8)
  before = dict(ops.fallbacks)
  y = ops.linear_forward("native", x, w, bias, True)
  _assert_exact(y, _on_grid(torch.relu(_gemm_ref("nt", x, w) + bias.double())), "linear forward")
  dy = _ints((batch, fout), 94, dtype)
  dym = dy.double() * (y > 0).double()
  stride = fout * fin + fout + 5
  rows = torch.full((groups, stride), SENTINEL, device="cuda")
  gw, gb = rows[0, :fout * fin].view(fout, fin), rows[0, fout * fin:fout * fin + fout]
  dx = ops.linear_backward("native", dy, x, w, y, True, True, gw, gb, groups, stride)
  assert ops.fallbacks == before
  per = batch // groups
  for g in range(groups):
    _assert_exact(rows[g, :fout * fin].view(fout, fin), _on_grid(_gemm_ref("tn", dym[g * per:(g + 1) * per], x[g * per:(g + 1) * per])), "linear wgrad %d" % g)
    _assert_exact(rows[g, fout * fin:fout * fin + fout].view(1, -1), _on_grid(dym[g * per:(g + 1) * per].sum(dim=0, keepdim=True)), "linear bias grad %d" % g)
  assert bool((rows[:, fout * fin + fout:] == SENTINEL).all())
  _assert_exact(dx, _on_grid(_gemm_ref("nn", dym, w)), "linear dgrad")


# ---------------------------------------------------------------------------- #
# Precision probes

@gpu
@pytest.mark.parametrize("layout", ["nt", "nn", "tn"])
@pytest.mark.parametrize("dyadic_side", ["a", "b"])
def test_tf32_operands_keep_eleven_bits(layout, dyadic_side):
  """Dyadic operands m * 2^-10 (exact in TF32, mostly not in bf16) against a +-1 operand with two non-zeros per output: the TF32 path
  must reproduce them exactly. Fails if either operand is handled at bf16 precision."""
  from aggregathor_b200.ops import nn_native as nat
  m, n, k = 257, 129, 1000
  sa, sb = _gemm_shapes(layout, m, n, k)
  # the sparse side has its non-zeros along K, per output row (A) or output column (B)
  a_kdim, b_kdim = (1 if layout in ("nt", "nn") else 0), (1 if layout == "nt" else 0)
  if dyadic_side == "a":
    a, b = _dyadic(sa, 101), _sparse_signs(sb, 102, b_kdim, FP32)
  else:
    a, b = _sparse_signs(sa, 103, a_kdim, FP32), _dyadic(sb, 104)
  dyadic = a if dyadic_side == "a" else b
  assert float((dyadic.to(BF16).float() != dyadic).float().mean()) > 0.6
  ref = _on_grid(_gemm_ref(layout, a, b), 2.0 ** -10)
  for bn in (64, 128):
    for splits in ((1, 3, None) if layout == "tn" else (1,)):
      what = "%s dyadic %s bn=%d splits=%s" % (layout, dyadic_side, bn, splits)
      if layout == "tn":
        out = nat.mm_tn(a, b, splits=splits, bn=bn)
      else:
        out = (nat.mm_nt if layout == "nt" else nat.mm_nn)(a, b, bn=bn)
      _assert_exact(out, ref, what)


def _tf32_truncated(t):
  """The top 19 bits of fp32 values (sign, exponent, 10 mantissa bits): what the tensor core reads of a TF32 operand."""
  return (t.view(torch.int32) & -8192).view(torch.float32)   # -8192 == 0xffffe000 as int32


@gpu
@pytest.mark.parametrize("layout", ["nt", "nn", "tn"])
def test_tf32_operand_truncation(layout):
  """Operands +-2^e * (1 + f * 2^-10), f in {0.25, 0.5, 0.75}: below TF32's last bit, so truncation reads +-2^e and round-to-nearest would
  not (f = 0.75 rounds up). The kernel result must equal the float64 product of the bit-masked operands, as the comment on `ElemTF32`
  states."""
  from aggregathor_b200.ops import nn_native as nat
  m, n, k = 200, 136, 128
  sa, sb = _gemm_shapes(layout, m, n, k)

  def probe(shape, seed):
    gen = _gen(seed)
    sign = torch.randint(0, 2, shape, generator=gen).double() * 2 - 1
    scale = 2.0 ** torch.randint(-1, 2, shape, generator=gen).double()
    frac = torch.tensor([0.25, 0.5, 0.75], dtype=torch.float64)[torch.randint(0, 3, shape, generator=gen)]
    return (sign * scale * (1 + frac * 2.0 ** -10)).float().cuda()

  a, b = probe(sa, 111), probe(sb, 112)
  ref = _on_grid(_gemm_ref(layout, _tf32_truncated(a), _tf32_truncated(b)), 2.0 ** -2)
  for bn in (64, 128):
    for splits in ((1, 2) if layout == "tn" else (1,)):
      if layout == "tn":
        out = nat.mm_tn(a, b, splits=splits, bn=bn)
      else:
        out = (nat.mm_nt if layout == "nt" else nat.mm_nn)(a, b, bn=bn)
      _assert_exact(out, ref, "%s bn=%d splits=%d (truncated operands)" % (layout, bn, splits))


@gpu
@pytest.mark.parametrize("dtype", [BF16, FP32], ids=["bf16", "tf32"])
@pytest.mark.parametrize("layout", ["nt", "nn", "tn"])
def test_random_data_error_bound(layout, dtype):
  """randn operands (bf16-rounded on the bf16 path): |C - C64| <= K 2^-23 (|A| @ |B|) element-wise, plus 2^-9 (|A| @ |B|) for the
  truncation of both TF32 operands. Prints the largest observed ratio of error to bound."""
  from aggregathor_b200.ops import nn_native as nat
  worst = 0.0
  for m, n, k in ((257, 129, 4096), (1000, 1000, 1000), (7, 300, 100352 // 4)):
    sa, sb = _gemm_shapes(layout, m, n, k)
    gen = torch.Generator(device="cuda").manual_seed(m + n)
    a = torch.randn(sa, device="cuda", generator=gen).to(dtype)
    b = torch.randn(sb, device="cuda", generator=gen).to(dtype)
    ref = _gemm_ref(layout, a, b)
    magnitude = _gemm_ref(layout, a.abs(), b.abs())
    bound = k * 2.0 ** -23 * magnitude
    if dtype == FP32:
      bound = bound + 2.0 ** -9 * magnitude
    for splits in ((1, 3, None) if layout == "tn" else (1,)):
      if layout == "tn":
        out = nat.mm_tn(a, b, splits=splits)
      else:
        out = (nat.mm_nt if layout == "nt" else nat.mm_nn)(a, b, out_dtype=FP32)
      err = (out.double() - ref).abs()
      ratio = float((err / bound).max())
      worst = max(worst, ratio)
      assert bool((err <= bound).all()), ("error above the bound", layout, dtype, m, n, k, splits, ratio)
  print("error / bound, %s %s: %.3e" % (layout, "bf16" if dtype == BF16 else "tf32", worst))


@gpu
def test_long_k_ternary_weight_gradient():
  """K = 100352 (a 56 x 56 x 32 batch of pixels) in one TN product: ternary operands keep every partial sum exact; split-K
  spreads the k-blocks over many CTAs."""
  from aggregathor_b200.ops import nn_native as nat
  k = 100352
  for dtype in (BF16, FP32):
    a, b = _ternary((k, 64), 121, dtype), _ternary((k, 72), 122, dtype)
    ref = _on_grid(_gemm_ref("tn", a, b))
    for splits in (1, None, 64):
      _assert_exact(nat.mm_tn(a, b, splits=splits), ref, "%s splits=%s" % (dtype, splits))

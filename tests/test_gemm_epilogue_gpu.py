"""Staged (shared memory + TMA store / reduce) and register epilogues of the Hopper GEMM and implicit-convolution kernels.

Operands are small integers, so every sum is exact in fp32 whatever order the kernel adds in (split-K reductions included): both
epilogues must produce the float64 oracle's value (bf16: its round-to-nearest-even), hence the same bits.
"""

import contextlib

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
BF16, FP32 = torch.bfloat16, torch.float32
SENTINEL = -777.0


def _nat():
  from aggregathor_b200.ops import nn_native
  return nn_native


@contextlib.contextmanager
def _epilogue(mode):
  _nat().set_gemm_epilogue(mode)
  try:
    yield
  finally:
    _nat().set_gemm_epilogue("staged")


def _ints(shape, seed, dtype, lo=-2, hi=2):
  gen = torch.Generator().manual_seed(seed)
  return torch.randint(lo, hi + 1, tuple(shape), generator=gen).to(dtype).cuda()


def _both(run):
  """`run()` under the register and the staged epilogue; asserts bit-identical results and returns them."""
  with _epilogue("regs"):
    regs = run()
  with _epilogue("staged"):
    staged = run()
  torch.cuda.synchronize()
  assert regs.dtype == staged.dtype and regs.shape == staged.shape
  assert torch.equal(regs.view(torch.int16 if regs.dtype == BF16 else torch.int32), staged.view(torch.int16 if staged.dtype == BF16 else torch.int32))
  return staged


def _expect(out, ref):
  ref = ref.to(out.dtype).cpu() if out.dtype == BF16 else ref.cpu()
  assert torch.equal(out.cpu().to(torch.float64), ref.to(torch.float64))


# ---------------------------------------------------------------------------- #
# GEMM

@pytest.mark.parametrize("dtype", [BF16, FP32], ids=["bf16", "tf32"])
@pytest.mark.parametrize("m,n,k", [(256, 1000, 2048), (300, 200, 64), (1000, 256, 130), (128, 64, 576)])
def test_gemm_modes_identical(dtype, m, n, k):
  """Forward (bias + ReLU, N not a multiple of the tile: the 1000-class FC layer), data gradient, split-K weight gradient."""
  nat = _nat()
  x, w, b = _ints((m, k), 1, dtype), _ints((n, k), 2, dtype), _ints((n,), 3, FP32)
  ref = (x.double() @ w.double().T + b.double()).clamp_min(0)
  _expect(_both(lambda: nat.mm_nt(x, w, bias=b, relu=True).clone()), ref)
  dy = _ints((m, n), 4, dtype)
  _expect(_both(lambda: nat.mm_nn(dy, w).clone()), dy.double() @ w.double())
  for splits in (1, 3):
    _expect(_both(lambda: nat.mm_tn(dy, x, splits=splits)), dy.double().T @ x.double())


def test_gemm_fp32_output_from_bf16():
  nat = _nat()
  x, w = _ints((384, 192), 5, BF16), _ints((520, 192), 6, BF16)
  _expect(_both(lambda: nat.mm_nt(x, w, out_dtype=FP32).clone()), x.double() @ w.double().T)


def test_bf16_output_rounds_ties_to_even():
  """Integers 256..1279 need 9-11 significant bits: every odd one is a tie or a near-tie for bf16's 8."""
  nat = _nat()
  m = 1024
  x = torch.zeros((m, 64), dtype=BF16, device="cuda")
  x[:, 0] = 256
  index = torch.arange(m, device="cuda")
  for c in range(5):   # row i: 256 + i as a sum of bf16-exact parts of at most 255
    x[:, 1 + c] = (index - 255 * c).clamp(0, 255).to(BF16)
  w = torch.zeros((72, 64), dtype=BF16, device="cuda")
  w[:, :6] = 1
  ref = x.double() @ w.double().T
  assert ref[:, 0].unique().numel() == m   # every value 256 .. 1279 once
  _expect(_both(lambda: nat.mm_nt(x, w).clone()), ref)


@pytest.mark.parametrize("dtype", [BF16, FP32], ids=["bf16", "tf32"])
@pytest.mark.parametrize("splits", [1, 4])
def test_grouped_split_k_leaves_guards_untouched(dtype, splits):
  """Per-worker weight gradients written into a flat buffer: every group's slice lands in place, the guard values around it stay."""
  nat = _nat()
  groups, m, n, kg, gap = 3, 200, 136, 96, 24
  stride = m * n + gap
  x, y = _ints((groups * kg, m), 7, dtype), _ints((groups * kg, n), 8, dtype)

  def run():
    flat = torch.full((16 + groups * stride,), SENTINEL, dtype=FP32, device="cuda")
    out = flat[16:16 + m * n].view(m, n)
    nat.mm_tn(x, y, out=out, splits=splits, groups=groups, group_stride=stride)
    return flat

  flat = _both(run).cpu()
  assert torch.all(flat[:16] == SENTINEL)
  for g in range(groups):
    base = 16 + g * stride
    ref = x[g * kg:(g + 1) * kg].double().T @ y[g * kg:(g + 1) * kg].double()
    _expect(flat[base:base + m * n].view(m, n), ref)
    assert torch.all(flat[base + m * n:base + stride] == SENTINEL)


@pytest.mark.parametrize("dtype", [BF16, FP32], ids=["bf16", "tf32"])
def test_dependent_chain_under_pdl(dtype):
  """Each product reads the previous one's output straight away (programmatic dependent launch): TMA stores must be complete."""
  nat = _nat()
  x = _ints((512, 128), 9, dtype, -1, 1)
  ws = [_ints((128, 128), 10 + i, dtype, -1, 1) for i in range(2)]   # |values| stay <= 128 * 128: exact in fp32, TF32 inputs <= 128
  eye = torch.eye(128, dtype=dtype, device="cuda")

  def run():
    h = x
    for w in ws:
      h = nat.mm_nt(h, eye)   # a copy through the GEMM: one more dependent launch per stage
      h = nat.mm_nt(h, w)
    return h.clone()

  out = _both(run)
  ref = x.double()
  for w in ws:
    ref = ref @ w.double().T
    ref = ref.to(dtype).double()   # bf16 intermediates round at each stage, as the kernel's outputs do
  _expect(out, ref)


# ---------------------------------------------------------------------------- #
# Implicit convolution

def _conv_refs(x, w, dy, stride, pads):
  """float64 fwd / dgrad / wgrad of NHWC x, [Cout, k, k, Cin] w, NHWC dy."""
  xd = x.double().cpu().permute(0, 3, 1, 2).requires_grad_(True)
  wd = w.double().cpu().permute(0, 3, 1, 2).requires_grad_(True)
  y = F.conv2d(F.pad(xd, (pads[2], pads[3], pads[0], pads[1])), wd, stride=stride)
  y.backward(dy.double().cpu().permute(0, 3, 1, 2))
  return y.detach().permute(0, 2, 3, 1), xd.grad.permute(0, 2, 3, 1), wd.grad.permute(0, 2, 3, 1)


# (n, hw, cin, cout, stride): pixel boxes 8x8x2 (56), 4x4x8 (28), 2x2x32 (14), 7x1x16 (7: 112-row box, register epilogue);
# stride 2: all four pixel parities of the data gradient
CONV_CASES = [(2, 56, 64, 64, 1), (8, 28, 64, 128, 1), (32, 14, 128, 64, 1), (16, 7, 64, 64, 1), (8, 28, 64, 64, 2), (32, 14, 64, 128, 2)]


@pytest.mark.parametrize("dtype", [BF16, FP32], ids=["bf16", "tf32"])
@pytest.mark.parametrize("n,hw,cin,cout,stride", CONV_CASES)
def test_implicit_conv_identical(dtype, n, hw, cin, cout, stride):
  nat = _nat()
  k, pads = 3, (1, 1, 1, 1)
  oh = hw // stride
  x, w, dy = _ints((n, hw, hw, cin), 11, dtype), _ints((cout, k, k, cin), 12, dtype), _ints((n, oh, oh, cout), 13, dtype)
  bias = _ints((cout,), 14, FP32)
  y_ref, dx_ref, dw_ref = _conv_refs(x, w, dy, stride, pads)

  def fwd():
    y = torch.empty((n, oh, oh, cout), dtype=dtype, device="cuda")
    return nat._conv_implicit(0, x, w, y, n, hw, hw, oh, oh, cin, cout, k, stride, pads, bias=bias, relu=True)

  def dgrad():
    dx = torch.full((n, hw, hw, cin), SENTINEL, dtype=dtype, device="cuda")
    return nat._conv_implicit(1, dy, w, dx, n, hw, hw, oh, oh, cin, cout, k, stride, pads)

  _expect(_both(fwd), (y_ref + bias.double().cpu()).clamp_min(0))
  _expect(_both(dgrad), dx_ref)
  groups = 2
  per = n // groups
  for splits in (1, 3):
    def wgrad():
      size = cout * k * k * cin
      flat = torch.full((groups * (size + 8),), SENTINEL, dtype=FP32, device="cuda")
      out = flat[:size].view(cout, k * k * cin)
      for g in range(groups):
        flat[g * (size + 8):g * (size + 8) + size].zero_()
      nat._conv_implicit(2, dy, x, out, n, hw, hw, oh, oh, cin, cout, k, stride, pads, splits=splits, groups=groups, group_stride=size + 8)
      return flat

    flat = _both(wgrad).cpu()
    size = cout * k * k * cin
    for g in range(groups):
      _, _, ref = _conv_refs(x[g * per:(g + 1) * per], w, dy[g * per:(g + 1) * per], stride, pads)
      _expect(flat[g * (size + 8):g * (size + 8) + size].view(cout, k, k, cin), ref)
      assert torch.all(flat[g * (size + 8) + size:(g + 1) * (size + 8)] == SENTINEL)

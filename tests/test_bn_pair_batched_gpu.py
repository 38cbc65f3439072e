"""Statistics + apply pair of batch norm with per-worker groups (`native/op_nn/layers.cu`), at the shapes of batched workers.

The apply kernels run a grid per group, and the closing norm's backward takes its masked gradient from the statistics kernel
instead of masking dy again. Both leave every output unchanged, which these tests assert at groups = 8, for C = 64, 256 and
2048, with the rows of a group both a multiple of what one sweep of the grid covers and not (32 images of 7 x 7 pixels):

  * against pure-torch replicas of the kernels' per-element arithmetic, exactly: the masked gradient (dy or +0), dbeta (integer
    gradients: exact sums in any order), dx = fma(a, dy', b * x) + c0 from the coefficients the statistics kernel left, and
    y = relu(fma(x, scale, shift) + residual) from the forward's scale and shift (an fp32 fma is emulated in float64: the
    product of two fp32 values is exact there);
  * against the float64 oracles of `test_layers_oracle_gpu.py`, within the bounds derived there (dgamma included).
"""

import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import test_layers_oracle_gpu as oracle  # noqa: E402
from test_layers_oracle_gpu import DECAY, EPS, record, run_bn_case  # noqa: E402,F401  (record: fixture)

CL = torch.channels_last
BF16, FP32 = torch.bfloat16, torch.float32
GROUPS = 8
U = 4   # unroll of the apply loops (bf16)


def _sms():
  return torch.cuda.get_device_properties(0).multi_processor_count


def _rows_per_group(c, kind):
  """'sweep': the group's octets are a multiple of U grid sweeps (the grid of one group is its share of 8 CTAs per SM);
  'maps7': 32 images of 7 x 7 pixels (1568 rows, no such multiple)."""
  if kind == "maps7":
    return 32 * 49
  octets = c // 8
  share = _sms() * 8 // GROUPS
  stride = share * 256 - share * 256 % octets
  return U * stride // octets


def _fma32(a, b, c):
  """fp32 fma(a, b, c): the product of two fp32 values is exact in float64, the sum is rounded once to fp32 from there."""
  return (a.double() * b.double() + c.double()).float()


def _nhwc(t2d):
  return t2d.view(t2d.shape[0], t2d.shape[1], 1, 1)


def _grid(shape, lo, hi, seed, dtype):
  gen = torch.Generator(device="cpu").manual_seed(seed)
  return torch.randint(lo, hi + 1, shape, generator=gen).to(device="cuda", dtype=dtype)


def _randn(shape, seed, dtype):
  gen = torch.Generator(device="cpu").manual_seed(seed)
  return torch.randn(shape, generator=gen).to(device="cuda", dtype=dtype)


def _same(out, ref, what):
  out, ref = out.float().reshape(ref.shape), ref.float()
  bad = out != ref
  assert not bool(bad.any()), "%s: %d elements differ, first at %s: got %r, want %r" % (
    what, int(bad.sum()), bad.nonzero()[0].tolist(), float(out[tuple(bad.nonzero()[0])]), float(ref[tuple(bad.nonzero()[0])]))


CASES = [(c, kind) for c in (64, 256, 2048) for kind in ("sweep", "maps7")]
DTYPES = [BF16, FP32]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp32"])
@pytest.mark.parametrize("c,kind", CASES)
def test_pair_batched_matches_replica(c, kind, dtype):
  from aggregathor_b200.ops import nn_native
  nn_native.set_bn_fused(False)
  try:
    rpg = _rows_per_group(c, kind)
    rows = GROUPS * rpg
    x = _randn((rows, c), 1, dtype)
    res = _randn((rows, c), 2, dtype)
    gamma, beta = 1 + 0.25 * _randn((c,), 3, FP32), 0.5 * _randn((c,), 4, FP32)
    mm, mv = torch.zeros(c, device="cuda"), torch.ones(c, device="cuda")
    # -- forward pair, closing form (residual) and plain ReLU form
    for residual in (res, None):
      y, mean, rstd, coef = nn_native.batchnorm_forward(_nhwc(x), gamma, beta, mm, mv, DECAY, EPS, True, GROUPS, _nhwc(residual) if residual is not None else None,
                                                        coef=True)
      sc, sh = (t.reshape(GROUPS, 1, c) for t in coef)
      v = _fma32(x.float().reshape(GROUPS, rpg, c), sc, sh.expand(GROUPS, rpg, c))
      if residual is not None:
        v = v + residual.float().reshape(GROUPS, rpg, c)
      want = torch.where(v > 0, v, torch.zeros_like(v)).to(dtype)
      _same(y, want.reshape(rows, c), "y C=%d rows/group=%d %s residual=%d" % (c, rpg, dtype, residual is not None))
    # -- backward pair of the closing norm: y with exact zeros and negative values, integer gradients
    dy = _grid((rows, c), -4, 4, 5, dtype)
    ymask = _grid((rows, c), -2, 2, 6, dtype)
    grads = torch.zeros((2, GROUPS, c), device="cuda")
    dx, dmasked = nn_native.batchnorm_backward(_nhwc(dy), _nhwc(x), _nhwc(ymask), gamma, mean, rstd, True, grads[0, 0], grads[1, 0], GROUPS, c, want_masked=True)
    cf = nn_native._workspace(x.device, "bn_coef", 3 * GROUPS * c, FP32)[:3 * GROUPS * c].reshape(GROUPS, 1, c, 3).clone()
    g = torch.where(ymask.float() > 0, dy.float(), torch.zeros((), device="cuda"))
    what = "C=%d rows/group=%d %s" % (c, rpg, dtype)
    _same(dmasked, g.to(dtype), "masked dy " + what)
    assert not bool(torch.signbit(dmasked.float()[g == 0]).any()), "masked dy " + what + ": a masked element is not +0"
    _same(grads[1], g.reshape(GROUPS, rpg, c).double().sum(dim=1).float(), "dbeta " + what)
    gg, xg = g.reshape(GROUPS, rpg, c), x.float().reshape(GROUPS, rpg, c)
    want = _fma32(cf[..., 0], gg, cf[..., 1] * xg) + cf[..., 2]
    _same(dx, want.to(dtype).reshape(rows, c), "dx " + what)
  finally:
    nn_native.set_bn_fused(True)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp32"])
@pytest.mark.parametrize("c,kind", CASES)
def test_pair_batched_matches_oracle(record, monkeypatch, c, kind, dtype):
  """Closing form (residual forward, masked backward) and plain ReLU form, through the pair, against the float64 oracles.
  x is |x| + 1 of the oracle module's grid operands (integers 1..9, sums still exact): with 1568 rows per group a channel whose
  mean is exactly 0 would come out as about 4e-16 (the fp64 division by a group size that is not a power of two), which the
  forward's 1-ulp bound on the rounded mean does not allow at 0; the mean and its bound are not what these tests are about."""
  operands = oracle._bn_operands

  def positive(*args, **kwargs):
    x, gamma, beta = operands(*args, **kwargs)
    return x.abs() + 1, gamma, beta

  monkeypatch.setattr(oracle, "_bn_operands", positive)
  rows = GROUPS * _rows_per_group(c, kind)
  run_bn_case(record, rows, c, GROUPS, dtype, fused=False, relu=True, residual=True, masked=True, seed=70, expect=("pair", "pair"))
  run_bn_case(record, rows, c, GROUPS, dtype, fused=False, relu=True, residual=False, masked=False, seed=80, expect=("pair", "pair"))

"""Depthwise convolution and windowed average pooling kernels (`native/op_nn/depthwise.cu`) against float64 oracles.

Every oracle below is plain float64 code that spells out the semantics it asserts; `test_oracles_match_torch_float64` checks
them against torch's float64 operators without a GPU.

Operands come in two families:
  * grid operands: x and dy small integers, w multiples of 1/8, all exact in bf16, so every product and every partial sum is exact
    in fp32 whatever the order (atomics included). The forward, the data gradient and the weight gradient then equal the float64
    result rounded to bf16 (ties to even) or to fp32, bit for bit. Average-pool windows sum integers exactly; the only errors are
    the reciprocal of the divisor, its product and the final rounding.
  * random operands, bounded by gamma_n * sum|terms| plus half a bf16 ulp of the output, n the number of taps or positions summed.

Each native case runs through `ops.nn` with a recording proxy around the native library, asserting that the native kernels served
it (status 0) and that `ops.nn.fallbacks` did not grow; the shapes the Python gate refuses must reach no kernel at all.
"""

import math

import pytest
import torch
import torch.nn.functional as F

from aggregathor_b200.models.core import same_padding

CL = torch.channels_last
BF16, FP32, F64 = torch.bfloat16, torch.float32, torch.float64
U24 = 2.0 ** -24
gpu = pytest.mark.gpu


# ---------------------------------------------------------------------------- #
# float64 oracles (x, dy: [N, C, H, W]; w: [C, k, k, 1]; pads = (top, bottom, left, right))

def _out(size, k, s, lo, hi):
  return (size + lo + hi - k) // s + 1


def _taps(h, w, oh, ow, k, s, pads, device):
  """For every tap (kh, kw): the input rows / columns the outputs read and whether they lie inside the image."""
  t, _, l, _ = pads
  for kh in range(k):
    ih = torch.arange(oh, device=device) * s + kh - t
    for kw in range(k):
      iw = torch.arange(ow, device=device) * s + kw - l
      yield kh, kw, ih, iw, ((ih >= 0) & (ih < h))[:, None] & ((iw >= 0) & (iw < w))[None, :]


def depthwise_forward_ref(x, w, s, pads):
  """y[n, c, oh, ow] = sum over the taps (kh, kw) whose pixel (oh s + kh - top, ow s + kw - left) lies in the image of
  x[n, c, pixel] * w[c, kh, kw]. Taps in the padding are skipped, not multiplied by zero (0 * inf would be NaN)."""
  n, c, h, wd = x.shape
  k = w.shape[1]
  oh, ow = _out(h, k, s, pads[0], pads[1]), _out(wd, k, s, pads[2], pads[3])
  xf, wf = x.to(F64), w.to(F64)
  y = torch.zeros((n, c, oh, ow), dtype=F64, device=x.device)
  for kh, kw, ih, iw, inside in _taps(h, wd, oh, ow, k, s, pads, x.device):
    vals = xf[:, :, ih.clamp(0, h - 1)][:, :, :, iw.clamp(0, wd - 1)] * wf[:, kh, kw, 0].view(1, c, 1, 1)
    y = y + torch.where(inside, vals, torch.zeros_like(vals))
  return y


def depthwise_dgrad_ref(dy, w, shape, s, pads):
  """Scatter: every output (oh, ow) adds dy[n, c, oh, ow] * w[c, kh, kw] to the in-image pixel its tap (kh, kw) reads; pixels read
  by no window get 0."""
  n, c, h, wd = shape
  k = w.shape[1]
  oh, ow = dy.shape[2], dy.shape[3]
  dyf, wf = dy.to(F64), w.to(F64)
  dx = torch.zeros((n, c, h * wd), dtype=F64, device=dy.device)
  for kh, kw, ih, iw, inside in _taps(h, wd, oh, ow, k, s, pads, dy.device):
    flat = (ih[:, None] * wd + iw[None, :])[inside]
    dx.index_add_(2, flat, (dyf * wf[:, kh, kw, 0].view(1, c, 1, 1))[:, :, inside])
  return dx.reshape(n, c, h, wd)


def depthwise_wgrad_ref(dy, x, k, s, pads, groups):
  """dw[g, c, kh, kw] = sum over the images of group g (consecutive blocks of N / groups) and the outputs whose tap (kh, kw) is in
  the image of dy[n, c, oh, ow] * x[n, c, pixel]. Returns [groups, C, k, k]."""
  n, c, h, wd = x.shape
  oh, ow = dy.shape[2], dy.shape[3]
  dyf, xf = dy.to(F64), x.to(F64)
  dw = torch.zeros((groups, c, k, k), dtype=F64, device=x.device)
  for kh, kw, ih, iw, inside in _taps(h, wd, oh, ow, k, s, pads, x.device):
    vals = xf[:, :, ih.clamp(0, h - 1)][:, :, :, iw.clamp(0, wd - 1)] * dyf
    vals = torch.where(inside, vals, torch.zeros_like(vals))
    dw[:, :, kh, kw] = vals.reshape(groups, n // groups, c, oh, ow).sum(dim=(1, 3, 4))
  return dw


def avgpool_forward_ref(x, k, s, pads):
  """y[n, c, oh, ow] = (sum of the in-image pixels of the k x k window at (oh s - top, ow s - left)) / (their number); a window
  wholly in the padding gives 0."""
  n, c, h, wd = x.shape
  oh, ow = _out(h, k, s, pads[0], pads[1]), _out(wd, k, s, pads[2], pads[3])
  xf = x.to(F64)
  total = torch.zeros((n, c, oh, ow), dtype=F64, device=x.device)
  count = torch.zeros((oh, ow), dtype=F64, device=x.device)
  for _, _, ih, iw, inside in _taps(h, wd, oh, ow, k, s, pads, x.device):
    vals = xf[:, :, ih.clamp(0, h - 1)][:, :, :, iw.clamp(0, wd - 1)]
    total = total + torch.where(inside, vals, torch.zeros_like(vals))
    count = count + inside
  return total / count.clamp_min(1), count


def avgpool_backward_ref(dy, shape, k, s, pads):
  """Every output's dy / (its window's in-image count) goes to each in-image pixel of its window."""
  n, c, h, wd = shape
  oh, ow = dy.shape[2], dy.shape[3]
  count = sum(inside.to(F64) for _, _, _, _, inside in _taps(h, wd, oh, ow, k, s, pads, dy.device))
  g = dy.to(F64) / count.clamp_min(1)
  dx = torch.zeros((n, c, h * wd), dtype=F64, device=dy.device)
  for _, _, ih, iw, inside in _taps(h, wd, oh, ow, k, s, pads, dy.device):
    dx.index_add_(2, (ih[:, None] * wd + iw[None, :])[inside], g[:, :, inside])
  return dx.reshape(n, c, h, wd)


# ---------------------------------------------------------------------------- #
# Oracle self-check (no GPU)

def test_oracles_match_torch_float64():
  gen = torch.Generator().manual_seed(0)
  for (n, c, h, w), k, s, pads in (((2, 3, 9, 8), 3, 2, (0, 1, 1, 1)), ((2, 2, 7, 11), 5, 3, (2, 2, 1, 3)), ((3, 2, 2, 1), 7, 1, (3, 3, 3, 3)),
                                   ((1, 2, 6, 6), 2, 4, (0, 0, 0, 0)), ((2, 1, 10, 5), 15, 1, (7, 7, 7, 7))):
    x = torch.randn((n, c, h, w), generator=gen, dtype=F64).requires_grad_(True)
    wt = torch.randn((c, k, k, 1), generator=gen, dtype=F64).requires_grad_(True)
    t, b, l, r = pads
    want = F.conv2d(F.pad(x, (l, r, t, b)), wt.permute(0, 3, 1, 2), None, s, 0, 1, c)
    y = depthwise_forward_ref(x.detach(), wt.detach(), s, pads)
    torch.testing.assert_close(y, want.detach(), rtol=1e-12, atol=1e-12)
    dy = torch.randn(want.shape, generator=gen, dtype=F64)
    (want * dy).sum().backward(retain_graph=True)
    torch.testing.assert_close(depthwise_dgrad_ref(dy, wt.detach(), x.shape, s, pads), x.grad, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(depthwise_wgrad_ref(dy, x.detach(), k, s, pads, 1)[0], wt.grad[..., 0], rtol=1e-12, atol=1e-12)
    if n > 1:   # per-group weight gradients are the gradients of each group's images alone
      x.grad, wt.grad = None, None
      (want[n // 2:] * dy[n // 2:]).sum().backward()
      torch.testing.assert_close(depthwise_wgrad_ref(dy, x.detach(), k, s, pads, n)[n // 2:].sum(dim=0), wt.grad[..., 0], rtol=1e-12, atol=1e-12)
    # average pool: the window sums with a zero-padded input, the divisor from a padded map of ones
    xa = x.detach().clone().requires_grad_(True)
    sums = F.avg_pool2d(F.pad(xa, (l, r, t, b)), k, s, divisor_override=1)
    counts = F.avg_pool2d(F.pad(torch.ones((1, 1, h, w), dtype=F64), (l, r, t, b)), k, s, divisor_override=1)
    want = sums / counts.clamp_min(1)
    got, count = avgpool_forward_ref(xa.detach(), k, s, pads)
    torch.testing.assert_close(got, want.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(count, counts[0, 0], rtol=0, atol=0)
    dy = torch.randn(want.shape, generator=gen, dtype=F64)
    (want * dy).sum().backward()
    torch.testing.assert_close(avgpool_backward_ref(dy, xa.shape, k, s, pads), xa.grad, rtol=1e-12, atol=1e-12)
  # a stride above k leaves pixels that no window reads: zero gradient there
  dx = depthwise_dgrad_ref(torch.ones((1, 1, 2, 2), dtype=F64), torch.ones((1, 2, 2, 1), dtype=F64), (1, 1, 6, 6), 4, (0, 0, 0, 0))
  assert float(dx[0, 0, 2:4].abs().sum()) == 0 and float(dx[0, 0, :, 2:4].abs().sum()) == 0 and float(dx[0, 0, :2, :2].sum()) == 4
  # an infinite weight whose tap lies in the padding leaves the output finite; on a zero pixel in the image it gives NaN
  x = torch.tensor([[[[0.0, 1.0], [2.0, 3.0]]]], dtype=F64)
  wt = torch.zeros((1, 3, 3, 1), dtype=F64)
  wt[0, 0, 0, 0] = math.inf
  y = depthwise_forward_ref(x, wt, 1, (1, 1, 1, 1))
  assert torch.isnan(y[0, 0, 1, 1]) and torch.isfinite(y[0, 0, 0]).all() and torch.isfinite(y[0, 0, :, 0]).all()
  # a window wholly in the padding averages to 0
  got, count = avgpool_forward_ref(torch.ones((1, 1, 2, 2), dtype=F64), 2, 1, (3, 0, 0, 0))
  assert float(count[0, 0]) == 0 and float(got[0, 0, 0, 0]) == 0 and float(got[0, 0, -1, 0]) == 1


# ---------------------------------------------------------------------------- #
# Helpers

def _ulp(ref, dtype):
  mant = 7 if dtype == BF16 else 23
  _, e = torch.frexp(ref.abs().clamp_min(2.0 ** -126))
  return torch.ldexp(torch.ones_like(ref, dtype=F64), (e - 1 - mant).to(torch.int32))


def _check(out, ref, bound, what):
  """Non-finite exactly where the oracle is (NaN vs +-inf), every other element within `bound`."""
  out, ref = out.to(F64).reshape(ref.shape), ref.to(F64)
  for name, fo, fr in (("nan", torch.isnan(out), torch.isnan(ref)), ("+inf", out == math.inf, ref == math.inf), ("-inf", out == -math.inf, ref == -math.inf)):
    if not torch.equal(fo, fr):
      raise AssertionError("%s: %s pattern differs from the oracle at %s" % (what, name, (fo != fr).nonzero()[:4].tolist()))
  fin = torch.isfinite(ref)
  bound = torch.as_tensor(bound, dtype=F64, device=ref.device).expand_as(ref)
  err = torch.where(fin, (out - ref).abs(), torch.zeros_like(ref))
  bad = err > bound
  if bad.any():
    first = bad.nonzero()[0].tolist()
    raise AssertionError("%s: %d elements out of bound; first at %s: got %r, oracle %r, bound %.3g"
                         % (what, int(bad.sum()), first, float(out[tuple(first)]), float(ref[tuple(first)]), float(bound[tuple(first)])))


def _exact(out, ref, what):
  """Bit for bit against the float64 oracle rounded once to the output type (ties to even)."""
  _check(out, ref.to(out.dtype).to(F64) if out.dtype != F64 else ref, 0.0, what)


def _gen(seed):
  return torch.Generator(device="cpu").manual_seed(seed)


def _grid_x(shape, seed, lo=-4, hi=4):
  return torch.randint(lo, hi + 1, shape, generator=_gen(seed)).to(BF16).cuda().contiguous(memory_format=CL)


def _grid_w(c, k, seed):
  return (torch.randint(-16, 17, (c, k, k, 1), generator=_gen(seed)).to(F64) / 8).to(BF16).cuda()


def _rand_x(shape, seed):
  return torch.randn(shape, generator=_gen(seed)).to(BF16).cuda().contiguous(memory_format=CL)


def _same(h, w, k, s):
  return same_padding(h, k, s) + same_padding(w, k, s)


NATIVE = ("agb_depthwise_forward", "agb_depthwise_dgrad", "agb_depthwise_wgrad", "agb_avgpool2d_forward", "agb_avgpool2d_backward")


class _Recorder:
  """Stands in for the native library: forwards everything, records (entry point, status) of the depthwise / pool entry points."""

  def __init__(self, lib):
    self._lib = lib
    self.calls = []

  def __getattr__(self, name):
    fn = getattr(self._lib, name)
    if name not in NATIVE:
      return fn

    def call(*args):
      status = fn(*args)
      self.calls.append((name, status))
      return status
    return call


@pytest.fixture
def record(monkeypatch):
  from aggregathor_b200.ops import nn as ops
  from aggregathor_b200.ops import nn_native
  rec = _Recorder(nn_native._lib())
  monkeypatch.setattr(nn_native, "_lib", lambda: rec)
  rec.fallbacks = dict(ops.fallbacks)
  yield rec


def _served(rec, names):
  """The calls since the last check were exactly `names`, each with status 0, and no op fell back to torch."""
  from aggregathor_b200.ops import nn as ops
  assert rec.calls == [(n, 0) for n in names], rec.calls
  assert ops.fallbacks == rec.fallbacks, (ops.fallbacks, rec.fallbacks)
  rec.calls.clear()


def _forward(rec, x, w, s, pads):
  from aggregathor_b200.ops import nn as ops
  y = ops.depthwise_forward("native", x, w, s, pads)
  _served(rec, ["agb_depthwise_forward"])
  return y


def _backward(rec, dy, x, w, s, pads, groups=1, stride=None, fill=0.0, prezeroed=False):
  """dx and the [groups, stride] fp32 gradient buffer (filled with `fill` first; worker g's [C, k, k] slot starts at g * stride)."""
  from aggregathor_b200.ops import nn as ops
  from aggregathor_b200.ops import nn_native
  c, k = w.shape[0], w.shape[1]
  stride = stride or c * k * k
  buf = torch.full((groups, stride), fill, dtype=FP32, device="cuda")
  grad_w = buf[0, :c * k * k].view(c, k, k, 1)
  if prezeroed:
    nn_native._all_groups(grad_w, groups, stride).zero_()
    with nn_native.prezeroed_gradients():
      dx = ops.depthwise_backward("native", dy, x, w, s, pads, grad_w, groups, stride)
  else:
    dx = ops.depthwise_backward("native", dy, x, w, s, pads, grad_w, groups, stride)
  _served(rec, ["agb_depthwise_wgrad", "agb_depthwise_dgrad"])
  return dx, buf


def run_grid_case(rec, n, c, h, w, k, s, pads, groups=1, seed=0, what=""):
  """Forward, data gradient and per-worker weight gradient on grid operands: all three bit for bit."""
  x, wt = _grid_x((n, c, h, w), seed), _grid_w(c, k, seed + 1)
  what = "%s N=%d C=%d %dx%d k=%d s=%d pads=%s groups=%d" % (what, n, c, h, w, k, s, pads, groups)
  y = _forward(rec, x, wt, s, pads)
  _exact(y, depthwise_forward_ref(x, wt, s, pads), what + " forward")
  dy = _grid_x(tuple(y.shape), seed + 2)
  dw_ref = depthwise_wgrad_ref(dy, x, k, s, pads, groups)
  assert float(dw_ref.abs().max()) < 2 ** 24                    # every partial sum an exact fp32 integer
  dx, buf = _backward(rec, dy, x, wt, s, pads, groups)
  _exact(dx, depthwise_dgrad_ref(dy, wt, x.shape, s, pads), what + " dgrad")
  _exact(buf.reshape(groups, c, k, k), dw_ref, what + " wgrad")
  return x, wt, dy


def run_random_case(rec, n, c, h, w, k, s, pads, seed, what=""):
  """Random bf16 operands: products are exact in fp32 (8-bit significands), so the error is the fp32 additions, gamma_n of the
  sum of |terms| with n the taps / positions summed, plus the output rounding (half a bf16 ulp; the wgrad stays in fp32)."""
  x, wt = _rand_x((n, c, h, w), seed), (torch.randn((c, k, k, 1), generator=_gen(seed + 1)) * 0.3).to(BF16).cuda()
  what = "%s random N=%d C=%d %dx%d k=%d s=%d" % (what, n, c, h, w, k, s)
  gamma = lambda m: m * U24 / (1 - m * U24)
  y = _forward(rec, x, wt, s, pads)
  ref = depthwise_forward_ref(x, wt, s, pads)
  taps = depthwise_forward_ref(torch.ones_like(x[:1, :1]), torch.ones_like(wt[:1]), s, pads)
  _check(y, ref, gamma(taps) * depthwise_forward_ref(x.abs(), wt.abs(), s, pads) + 0.5 * _ulp(ref, BF16), what + " forward")
  dy = _rand_x(tuple(y.shape), seed + 2)
  dx, buf = _backward(rec, dy, x, wt, s, pads)
  ref = depthwise_dgrad_ref(dy, wt, x.shape, s, pads)
  readers = depthwise_dgrad_ref(torch.ones_like(dy[:1, :1]), torch.ones_like(wt[:1]), (1, 1, h, w), s, pads)
  _check(dx, ref, gamma(readers) * depthwise_dgrad_ref(dy.abs(), wt.abs(), x.shape, s, pads) + 0.5 * _ulp(ref, BF16), what + " dgrad")
  ref = depthwise_wgrad_ref(dy, x, k, s, pads, 1)
  positions = n * dy.shape[2] * dy.shape[3] + 4 * 132       # the per-slice chains plus one fp32 atomic per slice
  _check(buf.reshape(1, c, k, k), ref, gamma(positions) * depthwise_wgrad_ref(dy.abs(), x.abs(), k, s, pads, 1), what + " wgrad")


# ---------------------------------------------------------------------------- #
# Depthwise

@gpu
@pytest.mark.parametrize("k", [1, 3, 5, 7, 15])
@pytest.mark.parametrize("s", [1, 2, 3])
def test_depthwise_filter_sizes_and_strides(record, k, s):
  """Every filter size the kernels take (1..15) and strides 1-3 on an odd 13 x 10 map with TF SAME padding (asymmetric for even
  totals: top 0, bottom 1 at k = 2m + 1 / s = 2 on even sides), grid and random operands."""
  h, w = 13, 10
  run_grid_case(record, 2, 24, h, w, k, s, _same(h, w, k, s), seed=k * 10 + s, what="sizes")
  run_random_case(record, 2, 24, h, w, k, s, _same(h, w, k, s), seed=k * 10 + s + 500, what="sizes")


@gpu
@pytest.mark.parametrize("h,w", [(12, 9), (9, 12), (16, 14)])
def test_depthwise_asymmetric_same_padding(record, h, w):
  """Even and odd H != W with k = 3, s = 2: SAME pads 0 before and 1 after on even sides (one bottom row / right column of padding
  only), 1 / 1 on odd sides."""
  pads = _same(h, w, 3, 2)
  assert (pads[0], pads[1]) == ((0, 1) if h % 2 == 0 else (1, 1))
  run_grid_case(record, 3, 8, h, w, 3, 2, pads, seed=h + w, what="asymmetric")


@gpu
@pytest.mark.parametrize("k,s", [(2, 3), (3, 5), (1, 2)])
def test_depthwise_stride_above_k(record, k, s):
  """Stride above the filter (VALID): pixels that no window reads must get exactly 0 in dx."""
  h, w = 17, 16
  x, wt, dy = run_grid_case(record, 2, 16, h, w, k, s, (0, 0, 0, 0), seed=40 + s, what="stride>k")
  ref = depthwise_dgrad_ref(dy, wt, x.shape, s, (0, 0, 0, 0))
  read = depthwise_dgrad_ref(torch.ones_like(dy[:1, :1]), torch.ones_like(wt[:1]), (1, 1, h, w), s, (0, 0, 0, 0))[0, 0] > 0
  assert not bool(read.all()) and float(ref[:, :, ~read].abs().sum()) == 0


@gpu
@pytest.mark.parametrize("hw", [(1, 1), (2, 2), (1, 3)])
def test_depthwise_tiny_maps_under_k7(record, hw):
  """1 x 1, 2 x 2 and 1 x 3 maps under k = 7 (SAME pads 3): every window lies mostly in the padding."""
  h, w = hw
  run_grid_case(record, 4, 8, h, w, 7, 1, _same(h, w, 7, 1), seed=50 + h * w, what="tiny")
  run_grid_case(record, 4, 8, h, w, 7, 2, _same(h, w, 7, 2), seed=60 + h * w, what="tiny")


@gpu
@pytest.mark.parametrize("c,w", [(8, 5), (24, 11), (264, 7), (264, 8), (1024, 2), (1024, 3), (1024, 4)])
def test_depthwise_channels_and_row_widths(record, c, w):
  """C in {8, 24, 264, 1024} with OW * C / 8 octets below (231), at (256, 512) and just above (264, 384) a multiple of the 256 threads
  of a row CTA."""
  run_grid_case(record, 2, c, 5, w, 3, 1, _same(5, w, 3, 1), seed=70 + c + w, what="channels")


@gpu
@pytest.mark.parametrize("k,s", [(3, 1), (3, 2)])
def test_depthwise_split_launches(record, k, s):
  """N * OH and N * H above 65535 (grid.y = images x rows): tall, narrow maps (5000 x 3, C = 8) over 30 images, so the host splits
  both the forward and the data gradient into several launches with a partial last one."""
  n, h, w = 30, 5000, 3
  oh = -(-h // s)
  assert n * oh > 65535 and n * h > 65535 and n % (65535 // h) and n % (65535 // oh)
  run_grid_case(record, n, 8, h, w, k, s, _same(h, w, k, s), seed=80 + s, what="split")


@gpu
@pytest.mark.parametrize("groups", [1, 3, 16])
def test_depthwise_wgrad_groups(record, groups):
  """Per-worker weight gradients, one image per group: a 3 x 3 map (9 positions, fewer than the slices planned for ~4 CTAs per SM)
  and a 20 x 20 map (the positions split across slices and summed by fp32 atomics)."""
  for hw in (3, 20):
    run_grid_case(record, groups, 24, hw, hw, 3, 1, _same(hw, hw, 3, 1), groups=groups, seed=90 + groups + hw, what="groups")


@gpu
def test_depthwise_wgrad_stride_gaps_and_garbage(record):
  """group_stride above C k k, sentinels in the gaps: the kernels write the [C, k, k] slots and nothing else. A buffer full of
  garbage is overwritten outside `prezeroed_gradients`; inside it, after the caller zeroes the slots, the result is the same."""
  n, c, h, w, k, groups = 3, 16, 9, 7, 5, 3
  pads = _same(h, w, k, 1)
  x, wt = _grid_x((n, c, h, w), 100), _grid_w(c, k, 101)
  dy = _grid_x((n, c, h, w), 102)
  ref = depthwise_wgrad_ref(dy, x, k, 1, pads, groups)
  stride = c * k * k + 40
  results = []
  for fill, prezeroed in ((-3.0, False), (float("nan"), False), (12345.0, True)):
    dx, buf = _backward(record, dy, x, wt, 1, pads, groups, stride, fill, prezeroed)
    what = "wgrad fill=%r prezeroed=%d" % (fill, prezeroed)
    _exact(buf[:, :c * k * k].reshape(groups, c, k, k), ref, what)
    gap = buf[:, c * k * k:]
    assert bool((gap.isnan() if math.isnan(fill) else gap == fill).all()), what + ": wrote into the gap between worker rows"
    results.append(buf[:, :c * k * k].clone())
  assert torch.equal(results[0], results[2])


@gpu
def test_depthwise_nonfinite(record):
  """NaN and +-inf in x and in the weights: exactly the outputs whose in-image window holds them are non-finite; a weight of +-inf
  whose tap lies in the padding for a border output leaves that output finite (taps in the padding are skipped)."""
  n, c, h, w, k = 2, 16, 8, 9, 3
  pads = _same(h, w, k, 1)
  x, wt = _grid_x((n, c, h, w), 110), _grid_w(c, k, 111)
  x[0, 1, 3, 4] = float("nan")
  x[1, 2, 0, 0] = float("inf")
  x[1, 3, 7, 8] = float("-inf")
  wt[5, 0, 0, 0] = float("inf")                                 # top-left tap: in the padding for the first row and column
  wt[6, 2, 1, 0] = float("-inf")
  y = _forward(record, x, wt, 1, pads)
  ref = depthwise_forward_ref(x, wt, 1, pads)
  assert bool(torch.isfinite(ref[:, 5, 0]).all()) and not bool(torch.isfinite(ref[:, 5, 1:, 1:]).all())
  _exact(y, ref, "nonfinite forward")
  dy = _grid_x(tuple(y.shape), 112)
  dy[1, 7, 4, 4] = float("nan")
  dx, buf = _backward(record, dy, x, wt, 1, pads)
  _exact(dx, depthwise_dgrad_ref(dy, wt, x.shape, 1, pads), "nonfinite dgrad")
  _exact(buf.reshape(1, c, k, k), depthwise_wgrad_ref(dy, x, k, 1, pads, 1), "nonfinite wgrad")


@gpu
def test_depthwise_k16_refused(record):
  """k = 16 is above the kernels' limit: the native library answers status 301 (an error, not a silent fallback)."""
  from aggregathor_b200.ops import nn as ops
  x, wt = _grid_x((1, 8, 20, 20), 120), _grid_w(8, 16, 121)
  with pytest.raises(RuntimeError, match="status 301"):
    ops.depthwise_forward("native", x, wt, 1, _same(20, 20, 16, 1))
  assert record.calls == [("agb_depthwise_forward", 301)]


@gpu
@pytest.mark.parametrize("case", ["C%8", "fp32", "multiplier", "non-square"])
def test_depthwise_gate_refusals(record, case):
  """Shapes the Python gate refuses (C % 8 != 0, fp32 activations, channel multiplier 2, a 3 x 5 filter) fall back to torch: no
  native call, one more fallback per direction, and the torch result."""
  from aggregathor_b200.ops import nn as ops
  c, k = (12 if case == "C%8" else 16), 3
  x = _grid_x((2, c, 9, 9), 130)
  wt = _grid_w(c, k, 131)
  if case == "fp32":
    x, wt = x.float(), wt.float()
  elif case == "multiplier":
    wt = torch.cat([wt, wt * 0.5], dim=0)
  elif case == "non-square":
    wt = (torch.randint(-16, 17, (c, 3, 5, 1), generator=_gen(132)).to(F64) / 8).to(BF16).cuda()
  pads = (1, 1, 2, 2) if case == "non-square" else (1, 1, 1, 1)
  before = dict(ops.fallbacks)
  y = ops.depthwise_forward("native", x, wt, 1, pads)
  dy = torch.ones_like(y)
  grad_w = torch.zeros(wt.shape, dtype=FP32, device="cuda")
  ops.depthwise_backward("native", dy, x, wt, 1, pads, grad_w)
  assert record.calls == []
  assert ops.fallbacks.get("depthwise_forward", 0) == before.get("depthwise_forward", 0) + 1
  assert ops.fallbacks.get("depthwise_backward", 0) == before.get("depthwise_backward", 0) + 1
  assert y.shape == (2, wt.shape[0], 9, 9)


# ---------------------------------------------------------------------------- #
# Windowed average pool

def _pool(rec, x, k, s, pads):
  from aggregathor_b200.ops import nn as ops
  y = ops.avgpool2d_forward("native", x, k, s, pads)
  _served(rec, ["agb_avgpool2d_forward"])
  return y


def _pool_back(rec, dy, shape, k, s, pads):
  from aggregathor_b200.ops import nn as ops
  dx = ops.avgpool2d_backward("native", dy, shape, k, s, pads)
  _served(rec, ["agb_avgpool2d_backward"])
  return dx


def run_pool_case(rec, n, c, h, w, k, s, pads, seed, what=""):
  """Grid x in [-8, 8]: window sums are exact, the kernel multiplies them by the fp32 reciprocal of the in-image count (two roundings,
  2 u) and rounds to bf16 (half an ulp). Backward: each term dy * (1 / count) takes 2 u, the chain of at most k * k additions
  (k * k) u of the sum of |terms|, then half an ulp."""
  x = _grid_x((n, c, h, w), seed, -8, 8)
  what = "%s avgpool N=%d C=%d %dx%d k=%d s=%d pads=%s" % (what, n, c, h, w, k, s, pads)
  y = _pool(rec, x, k, s, pads)
  ref, count = avgpool_forward_ref(x, k, s, pads)
  _check(y, ref, 2 * U24 * ref.abs() + 0.5 * _ulp(ref, BF16), what + " forward")
  exact = (count == count.clamp_min(1)) & ((count.long() & (count.long() - 1)) == 0)   # power-of-two counts: bit-exact
  _exact(y[:, :, exact], ref[:, :, exact], what + " forward (power-of-two windows)")
  dy = _grid_x(tuple(y.shape), seed + 1, -8, 8)
  dx = _pool_back(rec, dy, x.shape, k, s, pads)
  ref = avgpool_backward_ref(dy, x.shape, k, s, pads)
  terms = avgpool_backward_ref(dy.abs(), x.shape, k, s, pads)
  _check(dx, ref, (k * k + 2) * U24 * terms + 0.5 * _ulp(ref, BF16), what + " backward")


@gpu
@pytest.mark.parametrize("k,s,padding", [(3, 1, "SAME"), (3, 2, "SAME"), (5, 3, "VALID"), (2, 2, "SAME"), (7, 1, "SAME"), (15, 2, "SAME"), (3, 5, "VALID")])
@pytest.mark.parametrize("hw", [(12, 9), (1, 1), (2, 2)])
def test_avgpool(record, k, s, padding, hw):
  """SAME / VALID windows on an even-by-odd map (asymmetric SAME pads), and 1 x 1 / 2 x 2 maps where k = 7 and 15 windows lie mostly
  in the padding (divisors 1..4); stride 5 > k reads some pixels in no window (their gradient is 0)."""
  h, w = hw
  if padding == "VALID" and (h < k or w < k):
    pytest.skip("no VALID window fits")
  pads = _same(h, w, k, s) if padding == "SAME" else (0, 0, 0, 0)
  run_pool_case(record, 2, 24, h, w, k, s, pads, seed=140 + k + s + h, what=padding)


@gpu
def test_avgpool_windows_in_the_padding(record):
  """Explicit pads as large as the window: whole windows in the padding average to 0, and the corner windows divide by 1."""
  run_pool_case(record, 1, 8, 3, 4, 2, 1, (2, 1, 2, 0), seed=150, what="padding-only windows")


@gpu
@pytest.mark.parametrize("c,w", [(264, 7), (264, 8), (1024, 2), (1024, 3)])
def test_avgpool_channels(record, c, w):
  """Row widths below, at and just above a multiple of the 256 threads (OW * C / 8 octets)."""
  run_pool_case(record, 2, c, 6, w, 3, 1, _same(6, w, 3, 1), seed=160 + c + w, what="channels")


@gpu
def test_avgpool_split_launches(record):
  """N * OH and N * H above 65535: the host splits both directions into launches with a partial last one."""
  n, h, w = 30, 5000, 3
  assert n % (65535 // h)
  run_pool_case(record, n, 8, h, w, 3, 1, _same(h, w, 3, 1), seed=170, what="split")


@gpu
def test_avgpool_nonfinite_and_refusals(record):
  """NaN / +-inf reach exactly the outputs whose in-image window holds them (forward) and the pixels of the windows of a non-finite
  dy (backward); fp32 and C % 8 != 0 reach no kernel and count one fallback."""
  from aggregathor_b200.ops import nn as ops
  k, s, h, w = 3, 2, 10, 9
  pads = _same(h, w, k, s)
  x = _grid_x((2, 16, h, w), 180, -8, 8)
  x[0, 1, 4, 4], x[1, 2, 0, 0], x[1, 3, 9, 8] = float("nan"), float("inf"), float("-inf")
  y = _pool(record, x, k, s, pads)
  ref, _ = avgpool_forward_ref(x, k, s, pads)
  _check(y, ref, 2 * U24 * ref.abs().nan_to_num(posinf=0, neginf=0) + 0.5 * _ulp(ref.nan_to_num(posinf=0, neginf=0), BF16), "avgpool nonfinite forward")
  dy = _grid_x(tuple(y.shape), 181, -8, 8)
  dy[0, 5, 2, 2], dy[1, 6, 0, 4] = float("nan"), float("-inf")
  dx = _pool_back(record, dy, x.shape, k, s, pads)
  ref = avgpool_backward_ref(dy, x.shape, k, s, pads)
  terms = avgpool_backward_ref(dy.abs(), x.shape, k, s, pads).nan_to_num(posinf=0)
  _check(dx, ref, (k * k + 2) * U24 * terms + 0.5 * _ulp(ref.nan_to_num(posinf=0, neginf=0), BF16), "avgpool nonfinite backward")
  for xin in (x.float(), _grid_x((2, 12, h, w), 182)):
    before = dict(ops.fallbacks)
    assert ops.avgpool2d_forward("native", xin, k, s, pads) is None
    assert ops.fallbacks.get("avgpool2d_forward", 0) == before.get("avgpool2d_forward", 0) + 1
  assert record.calls == []

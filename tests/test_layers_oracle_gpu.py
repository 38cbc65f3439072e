"""Memory-bound layer kernels (`native/op_nn/layers.cu`, `layernorm.cu`, the ReLU6 of `depthwise.cu`) against float64 oracles.

Every oracle below is plain float64 code that spells out the semantics it asserts; no fp32 library kernel serves as a reference.
`test_oracles_match_torch_float64` checks the oracles themselves against torch's float64 CPU operators, without a GPU.

Operands come in two families:
  * grid operands: small integers (and dyadic parameters), so that every partial sum is exact in fp32 and in the fp64 atomics
    whatever the summation order; sums and means are then asserted bit for bit (or to the one rounding the algorithm itself
    performs), and every other output within a bound derived next to its assert;
  * random operands with |mean| / std up to 64 (bf16) and 1000 (fp32), for the conditioning of the variance.

Batch-norm cases also assert WHICH implementation served them (single-launch kernel or statistics + apply pair) through a
recording proxy around the native library, and choose their shapes with a Python mirror of the host-side plan of
`launch_bn_fused` / `plan_sums`, so each case keeps testing the boundary it names when the envelope or the SM count changes.
"""

import math

import pytest
import torch
import torch.nn.functional as F

CL = torch.channels_last
BF16, FP32, F64 = torch.bfloat16, torch.float32, torch.float64
U24 = 2.0 ** -24                        # unit roundoff of fp32 (round to nearest)
EPS = float(torch.tensor(1e-5, dtype=FP32))
DECAY = float(torch.tensor(0.9, dtype=FP32))
gpu = pytest.mark.gpu


# ---------------------------------------------------------------------------- #
# float64 oracles (device-agnostic: the CPU test runs them on the CPU)

def bn_forward_ref(x, gamma, beta, moving_mean, moving_var, decay, eps, relu, groups, residual=None):
  """x [rows, C]; consecutive blocks of rows / groups rows are one group. Per group g and channel c, over the group's n rows:
  mean = sum(x) / n; var = sum((x - mean)^2) / n (biased, for normalising); rstd = 1 / sqrt(var + eps);
  y = relu?((x - mean) * rstd * gamma + beta (+ residual)), gamma None = 1 (slim `scale=False`), relu keeps NaN.
  Moving statistics follow the decay convention with the UNBIASED variance, and only group 0 updates them:
  m = decay * m + (1 - decay) * mean_0 ; v = decay * v + (1 - decay) * var_0 * n / (n - 1).
  Returns y, mean [groups * C], rstd [groups * C], new moving mean, new moving var."""
  rows, c = x.shape
  n = rows // groups
  xg = x.to(F64).reshape(groups, n, c)
  mean = xg.sum(dim=1) / n
  var = ((xg - mean[:, None]) ** 2).sum(dim=1) / n
  rstd = 1.0 / torch.sqrt(var + eps)
  scale = rstd * (gamma.to(F64) if gamma is not None else 1.0)
  y = ((xg - mean[:, None]) * scale[:, None] + beta.to(F64)).reshape(rows, c)
  if residual is not None:
    y = y + residual.to(F64)
  if relu:
    y = torch.where(y > 0, y, torch.where(torch.isnan(y), y, torch.zeros_like(y)))
  unbiased = var[0] * n / (n - 1) if n > 1 else var[0]
  mm = decay * moving_mean.to(F64) + (1 - decay) * mean[0]
  mv = decay * moving_var.to(F64) + (1 - decay) * unbiased
  return y, mean.reshape(-1), rstd.reshape(-1), mm, mv


def bn_backward_ref(dy, x, y, gamma, mean, rstd, groups):
  """With the SAVED statistics mean / rstd [groups * C]: the mask is (y > 0) (y None: no mask; NaN in y masks to 0);
  g = dy * mask; per group: dbeta = sum g, dgamma = sum g * xhat with xhat = (x - mean) * rstd;
  dx = gamma * rstd * (g - dbeta / n - xhat * dgamma / n). Returns dx, g (the gradient of a fused residual input),
  dgamma [groups, C], dbeta [groups, C]."""
  rows, c = x.shape
  n = rows // groups
  g = dy.to(F64)
  if y is not None:
    g = torch.where(y.to(F64) > 0, g, torch.zeros_like(g))
  gg = g.reshape(groups, n, c)
  mu, rs = mean.to(F64).reshape(groups, 1, c), rstd.to(F64).reshape(groups, 1, c)
  xhat = (x.to(F64).reshape(groups, n, c) - mu) * rs
  dbeta = gg.sum(dim=1)
  dgamma = (gg * xhat).sum(dim=1)
  gm = gamma.to(F64) if gamma is not None else 1.0
  dx = gm * rs * (gg - dbeta[:, None] / n - xhat * dgamma[:, None] / n)
  return dx.reshape(rows, c), g, dgamma, dbeta


def colsum_ref(dy, y, groups):
  """Per group, the column sums of dy (masked by y > 0 when y is given): [groups, C] (the bias gradients)."""
  g = dy.to(F64)
  if y is not None:
    g = torch.where(y.to(F64) > 0, g, torch.zeros_like(g))
  return g.reshape(groups, -1, g.shape[1]).sum(dim=1)


def layernorm_forward_ref(x, gamma, beta, eps):
  """Per row: mean, biased variance, rstd = 1 / sqrt(var + eps); y = (x - mean) * rstd * gamma + beta."""
  xf = x.to(F64)
  mean = xf.sum(dim=1) / xf.shape[1]
  var = ((xf - mean[:, None]) ** 2).sum(dim=1) / xf.shape[1]
  rstd = 1.0 / torch.sqrt(var + eps)
  return (xf - mean[:, None]) * rstd[:, None] * gamma.to(F64) + beta.to(F64), mean, rstd


def layernorm_backward_ref(dy, x, gamma, mean, rstd):
  """With the saved mean / rstd: xhat = (x - mean) * rstd, g = dy * gamma;
  dx = rstd * (g - mean_c(g) - xhat * mean_c(g * xhat)); dgamma = sum_rows dy * xhat; dbeta = sum_rows dy."""
  d, xf = dy.to(F64), x.to(F64)
  xhat = (xf - mean.to(F64)[:, None]) * rstd.to(F64)[:, None]
  g = d * gamma.to(F64)
  dx = rstd.to(F64)[:, None] * (g - g.mean(dim=1, keepdim=True) - xhat * (g * xhat).mean(dim=1, keepdim=True))
  return dx, (d * xhat).sum(dim=0), d.sum(dim=0)


def softmax_xent_ref(logits, labels, smoothing, groups):
  """Targets t = smoothing / K everywhere plus (1 - smoothing) at the label; logp = z - logsumexp(z) (max-shifted);
  loss[g] = mean over the group's rows of -sum_k t * logp; dlogits = (exp(logp) - t) / (rows per group)."""
  z = logits.to(F64)
  b, k = z.shape
  mx = z.max(dim=1, keepdim=True).values
  logp = z - (mx + torch.log(torch.exp(z - mx).sum(dim=1, keepdim=True)))
  t = torch.full_like(z, smoothing / k)
  t[torch.arange(b, device=z.device), labels.long().to(z.device)] += 1.0 - smoothing
  n = b // groups
  loss = (-(t * logp).sum(dim=1)).reshape(groups, n).sum(dim=1) / n
  return loss, (torch.exp(logp) - t) / n, t, logp


def _windows(x, k, s, pads):
  """[N, C, H, W] -> [N, C, k*k, OH, OW] float64 windows (row-major taps), padded with -inf."""
  t, b, l, r = pads
  xp = F.pad(x.to(F64), (l, r, t, b), value=float("-inf"))
  n, c = x.shape[:2]
  oh, ow = (xp.shape[2] - k) // s + 1, (xp.shape[3] - k) // s + 1
  return F.unfold(xp, k, stride=s).reshape(n, c, k * k, oh, ow)


def maxpool_forward_ref(x, k, s, pads):
  """-inf padding; the value is the window maximum and the index the FIRST maximal tap in row-major window order; a window
  holding NaN yields NaN and the index of its LAST NaN tap (the tap whose NaN is compared last, as torch's kernels do)."""
  win = _windows(x, k, s, pads)
  isnan = torch.isnan(win)
  taps = k * k
  first_max = torch.where(isnan, torch.full_like(win, float("-inf")), win).argmax(dim=2)   # torch.argmax: first maximal index
  last_nan = taps - 1 - isnan.flip(2).to(torch.uint8).argmax(dim=2)
  has_nan = isnan.any(dim=2)
  idx = torch.where(has_nan, last_nan, first_max)
  val = torch.where(has_nan, torch.full_like(win[:, :, 0], float("nan")), win.gather(2, first_max[:, :, None]).squeeze(2))
  return val, idx


def maxpool_backward_ref(dy, idx, shape, k, s, pads):
  """Each output's gradient goes to the input tap its window index names (taps in the padding are dropped)."""
  n, c, h, w = shape
  t, b, l, r = pads
  hp, wp = h + t + b, w + l + r
  oh, ow = idx.shape[2], idx.shape[3]
  rows = torch.arange(oh).view(oh, 1) * s + idx.cpu() // k
  cols = torch.arange(ow).view(1, ow) * s + idx.cpu() % k
  flat = (rows * wp + cols).reshape(n, c, -1).to(dy.device)
  dxp = torch.zeros((n, c, hp * wp), dtype=F64, device=dy.device).scatter_add_(2, flat, dy.to(F64).reshape(n, c, -1))
  return dxp.reshape(n, c, hp, wp)[:, :, t:t + h, l:l + w]


def avgpool_ref(x):
  """Global average pool: mean over H x W -> [N, C]."""
  return x.to(F64).mean(dim=(2, 3))


IMAGE_MODES = {"vgg": ((123.68, 116.78, 103.94), 1.0), "inception": ((127.5,) * 3, 1.0 / 127.5), "lenet": ((128.0,) * 3, 1.0 / 128.0)}


def image_normalize_ref(images, mode):
  """uint8 NHWC -> (x - mean[c]) * scale in float64, NHWC."""
  means, scale = IMAGE_MODES[mode]
  c = images.shape[-1]
  return (images.to(F64) - torch.tensor(means[:c], dtype=F64, device=images.device)) * scale


# ---------------------------------------------------------------------------- #
# Oracle self-check (no GPU)

def test_oracles_match_torch_float64():
  gen = torch.Generator().manual_seed(0)
  x = torch.randn((24, 16), generator=gen, dtype=F64) * 3 + 1
  gamma, beta = torch.rand(16, generator=gen, dtype=F64) + 0.5, torch.randn(16, generator=gen, dtype=F64)
  for groups in (1, 3):
    y, mean, rstd, mm, mv = bn_forward_ref(x, gamma, beta, torch.zeros(16, dtype=F64), torch.ones(16, dtype=F64), 0.9, 1e-3, False, groups)
    xs = x.reshape(groups, -1, 16)
    rm, rv = torch.zeros(16, dtype=F64), torch.ones(16, dtype=F64)
    want = [F.batch_norm(xs[g], rm if g == 0 else None, rv if g == 0 else None, gamma, beta, True, 0.1, 1e-3) for g in range(groups)]
    torch.testing.assert_close(y, torch.cat(want), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(mm, rm, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(mv, rv, rtol=1e-12, atol=1e-12)
    # backward through autograd, with a ReLU mask and a residual-free unit
    xr = x.clone().requires_grad_(True)
    gr = gamma.clone().requires_grad_(True)
    br = beta.clone().requires_grad_(True)
    out = torch.cat([F.batch_norm(xs_g, None, None, gr, br, True, 0.1, 1e-3) for xs_g in xr.reshape(groups, -1, 16)])
    dy = torch.randn(out.shape, generator=gen, dtype=F64)
    mask_src = torch.randn(out.shape, generator=gen, dtype=F64)
    mask_src[0, 0] = float("nan")
    (out * dy * (mask_src > 0)).sum().backward()
    dx, g, dgm, dbt = bn_backward_ref(dy, x, mask_src, gamma, mean, rstd, groups)
    torch.testing.assert_close(dx, xr.grad, rtol=1e-10, atol=1e-10)
    assert float(g[0, 0]) == 0.0
    if groups == 1:
      torch.testing.assert_close(dgm[0], gr.grad, rtol=1e-10, atol=1e-10)
      torch.testing.assert_close(dbt[0], br.grad, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(colsum_ref(dy, mask_src, groups).sum(dim=0), (dy * (mask_src > 0)).sum(dim=0), rtol=1e-12, atol=1e-12)
  # LayerNorm
  xl = (torch.randn((5, 40), generator=gen, dtype=F64) + 2).requires_grad_(True)
  y, mean, rstd = layernorm_forward_ref(xl.detach(), gamma.repeat(3)[:40], beta.repeat(3)[:40], 1e-5)
  gl, bl = gamma.repeat(3)[:40].clone().requires_grad_(True), beta.repeat(3)[:40].clone().requires_grad_(True)
  want = F.layer_norm(xl, (40,), gl, bl, 1e-5)
  torch.testing.assert_close(y, want.detach(), rtol=1e-12, atol=1e-12)
  dy = torch.randn(want.shape, generator=gen, dtype=F64)
  (want * dy).sum().backward()
  dx, dgm, dbt = layernorm_backward_ref(dy, xl.detach(), gl.detach(), mean, rstd)
  for a, b in ((dx, xl.grad), (dgm, gl.grad), (dbt, bl.grad)):
    torch.testing.assert_close(a, b, rtol=1e-10, atol=1e-10)
  # softmax cross-entropy with label smoothing, per-group means
  z = (torch.randn((12, 33), generator=gen, dtype=F64) * 20).requires_grad_(True)
  labels = torch.randint(0, 33, (12,), generator=gen)
  loss, dz, _, _ = softmax_xent_ref(z.detach(), labels, 0.1, 4)
  want = torch.stack([F.cross_entropy(z[3 * g:3 * g + 3], labels[3 * g:3 * g + 3], label_smoothing=0.1) for g in range(4)])
  torch.testing.assert_close(loss, want.detach(), rtol=1e-12, atol=1e-12)
  want.sum().backward()
  torch.testing.assert_close(dz, z.grad, rtol=1e-12, atol=1e-12)
  # max-pool: values and argmax against F.max_pool2d on an explicitly -inf padded input, ties and NaN included
  xm = torch.randint(-2, 3, (2, 3, 9, 8), generator=gen).to(F64)
  xm[0, 1, 4, 4] = float("nan")
  for k, s, pads in ((3, 2, (1, 1, 1, 1)), (2, 2, (0, 1, 1, 0)), (5, 2, (2, 1, 0, 2))):
    val, idx = maxpool_forward_ref(xm, k, s, pads)
    xp = F.pad(xm, (pads[2], pads[3], pads[0], pads[1]), value=float("-inf"))
    want, where = F.max_pool2d(xp, k, s, return_indices=True)
    assert torch.equal(torch.isnan(val), torch.isnan(want))
    torch.testing.assert_close(val.nan_to_num(), want.nan_to_num(), rtol=0, atol=0)
    wp = xp.shape[3]
    oh = torch.arange(val.shape[2]).view(-1, 1) * s
    ow = torch.arange(val.shape[3]).view(1, -1) * s
    assert torch.equal((where // wp - oh) * k + (where % wp - ow), idx)
    dy = torch.randint(-3, 4, val.shape, generator=gen).to(F64)
    xq = xp.clone().requires_grad_(True)
    F.max_pool2d(xq, k, s).backward(dy)
    torch.testing.assert_close(maxpool_backward_ref(dy, idx, xm.shape, k, s, pads), xq.grad[:, :, pads[0]:pads[0] + 9, pads[2]:pads[2] + 8], rtol=0, atol=0)
  torch.testing.assert_close(avgpool_ref(xm[1:]), F.adaptive_avg_pool2d(xm[1:], 1)[:, :, 0, 0], rtol=1e-12, atol=1e-12)
  img = torch.randint(0, 256, (2, 3, 4, 3), generator=gen, dtype=torch.uint8)
  for mode, want in (("vgg", img.to(F64) - torch.tensor([123.68, 116.78, 103.94], dtype=F64)), ("inception", img.to(F64) / 127.5 - 1), ("lenet", (img.to(F64) - 128) / 128)):
    torch.testing.assert_close(image_normalize_ref(img, mode), want, rtol=1e-12, atol=1e-12)


# ---------------------------------------------------------------------------- #
# Comparison helpers

def _ulp(ref, dtype):
  """One unit in the last place of each |ref| in `dtype` (bf16: 8 significant bits, fp32: 24), floored at the smallest normal."""
  mant = 7 if dtype == BF16 else 23
  _, e = torch.frexp(ref.abs().clamp_min(2.0 ** -126))
  return torch.ldexp(torch.ones_like(ref, dtype=F64), (e - 1 - mant).to(torch.int32))


def _check(out, ref, bound, what, rows_per_group=None):
  """Non-finite exactly where the oracle is (NaN vs +-inf), every other element within `bound` (a tensor or a number).
  For [rows, C] tensors, `rows_per_group` turns the first failing element into (group, row, channel)."""
  out, ref = out.to(F64).reshape(ref.shape), ref.to(F64)
  for name, fo, fr in (("nan", torch.isnan(out), torch.isnan(ref)), ("+inf", out == math.inf, ref == math.inf), ("-inf", out == -math.inf, ref == -math.inf)):
    if not torch.equal(fo, fr):
      where = (fo != fr).nonzero()[:4].tolist()
      raise AssertionError("%s: %s pattern differs from the oracle at %s" % (what, name, where))
  fin = torch.isfinite(ref)
  bound = torch.as_tensor(bound, dtype=F64, device=ref.device).expand_as(ref)
  err = torch.where(fin, (out - ref).abs(), torch.zeros_like(ref))
  bad = err > bound
  if bad.any():
    first = bad.nonzero()[0].tolist()
    place = "index %s" % (first,)
    if rows_per_group is not None and len(first) == 2:
      place = "group %d row %d channel %d" % (first[0] // rows_per_group, first[0], first[1])
    raise AssertionError("%s: %d elements out of bound; first at %s: got %r, oracle %r, bound %.3g (max err/bound %.3g)"
                         % (what, int(bad.sum()), place, float(out[tuple(first)]), float(ref[tuple(first)]), float(bound[tuple(first)]),
                            float((err / bound.clamp_min(1e-300)).max())))


def _exact(out, ref, what, rows_per_group=None):
  _check(out, ref, 0.0, what, rows_per_group)


def _grid(shape, lo, hi, seed, dtype, device="cuda"):
  gen = torch.Generator(device="cpu").manual_seed(seed)
  return torch.randint(lo, hi + 1, shape, generator=gen).to(device=device, dtype=dtype)


def _as_nhwc(t2d):
  """[rows, C] -> (rows, C, 1, 1) channels_last view of the same memory (what the batch-norm entry points take)."""
  return t2d.view(t2d.shape[0], t2d.shape[1], 1, 1)


# ---------------------------------------------------------------------------- #
# Host plan mirror and the recording proxy

SCRATCH_BYTES, MOVING_BYTES, STASH_BYTES = 512 * 16 * 4, 12 * 1024, 180 * 1024
MAX_PAIRS = 16384                        # (group, channel) pairs of one workspace half
DEFAULT_LIMITS = (72, 40, 4096)          # forward MB, backward MB, fewest rows


def _sms():
  return torch.cuda.get_device_properties(0).multi_processor_count


def fused_plan(rows, c, groups, bwd, extra, sms, limits=DEFAULT_LIMITS):
  """Mirror of `launch_bn_fused`: None when the single-launch kernel declines the shape, else its plan."""
  if c % 8 or 3 * c * 4 > SCRATCH_BYTES or c * 4 > MOVING_BYTES or groups < 1 or groups > sms or rows % groups or c * groups > MAX_PAIRS:
    return None
  fwd_mb, bwd_mb, min_rows = limits
  if rows < (min_rows // 4 if extra else min_rows) or rows * c * 2 > ((bwd_mb if bwd else fwd_mb) << 20):
    return None
  octets = c // 8
  rpg = rows // groups
  min_vecs = max(octets * 32, 2048)
  want = -(-rpg * octets // min_vecs)
  ctas = max(1, min(want, sms // groups))
  rows_per_cta = -(-rpg // ctas)
  replicas = min(max(1, min(MAX_PAIRS // (c * groups), 8)), ctas)
  stride = 512 - 512 % octets
  return dict(ctas_per_group=ctas, rows_per_cta=rows_per_cta, replicas=replicas, stash_vecs=STASH_BYTES // 16 // (2 if bwd else 1),
              lanes=stride // octets, empty_chunks=sum(1 for k in range(ctas) if k * rows_per_cta >= rpg))


def sums_plan(rpg, c, groups, sms):
  """Mirror of `plan_sums` (statistics kernel of the pair): rows per CTA and the number of row chunks."""
  strips = -(-(c // 8) // 8)
  target = max(1, -(-(sms * 6) // (strips * groups)))
  rows_per_cta = max(-(-rpg // target), 32 * 4)
  return dict(rows_per_cta=rows_per_cta, chunks=-(-rpg // rows_per_cta))


def _chain(plan, pair_plan):
  """Longest chain of fp32 additions behind one statistic: the per-thread partial plus the fixed-order fold over the row lanes."""
  if plan is not None:
    return -(-plan["rows_per_cta"] // plan["lanes"]) + plan["lanes"]
  return -(-pair_plan["rows_per_cta"] // 32) + 32


BN_ENTRIES = ("agb_bn_forward_fused", "agb_bn_backward_fused", "agb_bn_forward", "agb_bn_forward_f32", "agb_bn_backward", "agb_bn_backward_f32")
COVERAGE = set()


class _Recorder:
  """Stands in for the native library: forwards everything, records (entry point, status) of the batch-norm entry points."""

  def __init__(self, lib):
    self._lib = lib
    self.calls = []

  def __getattr__(self, name):
    fn = getattr(self._lib, name)
    if name not in BN_ENTRIES:
      return fn

    def call(*args):
      status = fn(*args)
      self.calls.append((name, status))
      return status
    return call


@pytest.fixture
def record(monkeypatch):
  from aggregathor_b200.ops import nn_native
  rec = _Recorder(nn_native._lib())
  monkeypatch.setattr(nn_native, "_lib", lambda: rec)
  yield rec
  nn_native.set_bn_fused(True)
  nn_native.set_bn_fused_limits(*DEFAULT_LIMITS)


def _served(rec, bwd):
  """'fused' or 'pair' for the last batch-norm call of the given direction (asserting the status protocol)."""
  direction = "backward" if bwd else "forward"
  name, status = [(n, s) for n, s in rec.calls if direction in n][-1]
  assert status == 0, (name, status)
  return "fused" if name.endswith("_fused") else "pair"


# ---------------------------------------------------------------------------- #
# Batch norm

def _bn_operands(rows, c, groups, dtype, seed, gamma_on=True):
  x = _grid((rows, c), -8, 8, seed, dtype)
  gamma = _grid((c,), 2, 6, seed + 1, FP32) / 4 if gamma_on else None       # dyadic: exact in fp32
  beta = _grid((c,), -4, 4, seed + 2, FP32) / 8
  return x, gamma, beta


def _y_bound(x, scale, shift_parts, extra, ref, dtype, rstd_rel):
  """Bound on a forward output. The kernels compute v = x * scale + shift (+ residual) in fp32 from scale = gamma * rstd and
  shift = beta - float(mean) * gamma * rstd: with rstd within `rstd_rel` and at most 6 further fp32 roundings (mean to fp32,
  two products, a difference, the fma, the residual add), |v - exact| <= (rstd_rel + 6 u) * (|x scale| + |beta| +
  |mean scale| + |residual|) (`shift_parts` = |beta| + |mean scale|: the rounding errors of the shift scale with its parts, not
  with the shift); rounding v to the output type adds at most one half ulp, taken as one ulp of the oracle (v may cross into the
  next binade)."""
  terms = (x.to(F64) * scale).abs() + shift_parts + (extra.to(F64).abs() if extra is not None else 0)
  return _ulp(ref, dtype) + (rstd_rel + 6 * U24) * terms


def _bn_forward(rec, x, gamma, beta, mm, mv, relu, groups, residual):
  from aggregathor_b200.ops import nn_native
  out = nn_native.batchnorm_forward(_as_nhwc(x), gamma, beta, mm, mv, DECAY, EPS, relu, groups, _as_nhwc(residual) if residual is not None else None)
  assert out is not None
  y, mean, rstd = out
  return y.reshape(x.shape), mean, rstd, _served(rec, False)


def run_bn_case(rec, rows, c, groups, dtype=BF16, fused=True, relu=True, residual=False, gamma_on=True, masked=False, seed=0, limits=DEFAULT_LIMITS,
                expect=None, tags=()):
  """One forward + backward on grid operands against the oracles; returns the two paths that served them."""
  from aggregathor_b200.ops import nn_native
  sms = _sms()
  nn_native.set_bn_fused(fused)
  nn_native.set_bn_fused_limits(*limits)
  x, gamma, beta = _bn_operands(rows, c, groups, dtype, seed, gamma_on)
  res = _grid((rows, c), -3, 3, seed + 3, dtype) if residual else None
  mm0, mv0 = _grid((c,), -2, 2, seed + 4, FP32), _grid((c,), 1, 4, seed + 5, FP32)
  mm, mv = mm0.clone(), mv0.clone()
  rpg = rows // groups
  # -- forward
  fplan = fused_plan(rows, c, groups, False, residual, sms, limits) if (fused and dtype == BF16) else None
  y, mean, rstd, path = _bn_forward(rec, x, gamma, beta, mm, mv, relu, groups, res)
  assert path == ("fused" if fplan else "pair"), (path, fplan)
  if expect is not None:
    assert path == expect[0], ("forward", path, expect)
  COVERAGE.add(("forward", path, str(dtype)))
  for tag in tags:
    COVERAGE.add(("forward", path) + tag)
  yr, mr, rr, mmr, mvr = bn_forward_ref(x, gamma, beta, mm0, mv0, DECAY, EPS, relu, groups, res)
  what = "bn forward %s C=%d rows=%d groups=%d %s relu=%d res=%d gamma=%d" % (path, c, rows, groups, dtype, relu, residual, gamma_on)
  # every partial sum is an exact integer (|x| <= 8, squares <= 64, far below 2^24 in any fp32 chain); the mean is one division
  # (exact when n is a power of two) plus the pivot, rounded once to fp32: bit-exact vs the rounded oracle when n = 2^k, else <= 1 ulp
  pow2 = rpg & (rpg - 1) == 0
  _check(mean, mr.to(FP32), 0.0 if pow2 else _ulp(mr, FP32), what + " save_mean")
  # rstd = rsqrtf(float(var) + eps): var to fp32 and the eps add are two roundings (2 u on the argument, 1 u on the result), and
  # rsqrtf is within 2 ulp (CUDA math accuracy tables): 2 ulp + 1 u <= 5 u <= 2^-21 relative
  _check(rstd, rr, 2.0 ** -21 * rr, what + " save_rstd")
  gm = gamma.to(F64) if gamma is not None else torch.ones(c, dtype=F64, device="cuda")
  scale = (rr.reshape(groups, c) * gm).repeat_interleave(rpg, dim=0)
  shift = beta.to(F64).abs() + (mr.reshape(groups, c) * rr.reshape(groups, c) * gm).abs().repeat_interleave(rpg, dim=0)
  _check(y, yr, _y_bound(x, scale, shift, res, yr, dtype, 2.0 ** -21), what + " y", rpg)
  # moving statistics: the mean and the unbiased variance rounded to fp32, then decay * m + (1 - decay) * s: (1 - decay) is exact
  # (Sterbenz), three more roundings (two products and the sum): <= 4 u of |decay m| + |(1 - decay) s|
  _check(mm, mmr, 4 * U24 * (DECAY * mm0.to(F64).abs() + (1 - DECAY) * mr[:c].abs()) + 1e-300, what + " moving_mean")
  n = rpg
  _check(mv, mvr, 4 * U24 * (DECAY * mv0.to(F64).abs() + (1 - DECAY) * (mvr - DECAY * mv0.to(F64)).abs() / (1 - DECAY)) + 1e-300, what + " moving_var")
  # -- backward: the saved statistics of the oracle, rounded to fp32, are its inputs
  dy = _grid((rows, c), -4, 4, seed + 6, dtype)
  ymask = _grid((rows, c), -2, 2, seed + 7, dtype) if relu else None
  if ymask is not None:
    ymask[rows // 2, c - 1] = float("nan")                       # a NaN mask entry masks to zero
  smean, srstd = mr.to(FP32), rr.to(FP32)
  stride = c + 8
  sentinel = 12345.0
  grads = torch.full((groups, 2, stride), sentinel, dtype=FP32, device="cuda")
  bplan = fused_plan(rows, c, groups, True, masked and relu, sms, limits) if (fused and dtype == BF16) else None
  out = nn_native.batchnorm_backward(_as_nhwc(dy), _as_nhwc(x), _as_nhwc(ymask) if ymask is not None else None, gamma, smean, srstd, relu,
                                     grads[0, 0, :c] if gamma_on else None, grads[0, 1, :c], groups, grads.stride(0), want_masked=masked and relu)
  dx, dmask = out if (masked and relu) else (out, None)
  bpath = _served(rec, True)
  assert bpath == ("fused" if bplan else "pair"), (bpath, bplan)
  if expect is not None:
    assert bpath == expect[1], ("backward", bpath, expect)
  COVERAGE.add(("backward", bpath, str(dtype)))
  for tag in tags:
    COVERAGE.add(("backward", bpath) + tag)
  dxr, gr, dgr, dbr = bn_backward_ref(dy, x, ymask, gamma, smean, srstd, groups)
  what = "bn backward %s C=%d rows=%d groups=%d %s relu=%d masked=%d gamma=%d" % (bpath, c, rows, groups, dtype, relu, masked, gamma_on)
  untouched = grads[:, :, c:]
  assert bool((untouched == sentinel).all()), what + ": wrote outside the [groups, C] gradient slots"
  if not gamma_on:
    assert bool((grads[:, 0, :c] == sentinel).all()), what + ": wrote dgamma without gamma"
  _exact(grads[:, 1, :c], dbr, what + " dbeta")                  # sums of integers: exact in any order
  # dgamma: each term dy' * ((x - mu) * rs) takes at most 3 roundings, then one fp32 chain of L additions (per-thread partial +
  # fold; the fp64 atomics add exactly) and one rounding to fp32: |err| <= (L + 3) u * sum|dy' xhat| + u |dgamma|
  chain = _chain(bplan, sums_plan(rpg, c, groups, sms))
  gx = (gr.reshape(groups, rpg, c) * ((x.to(F64).reshape(groups, rpg, c) - smean.to(F64).reshape(groups, 1, c)) * srstd.to(F64).reshape(groups, 1, c))).abs().sum(dim=1)
  dg_bound = (chain + 3) * U24 * gx + U24 * dgr.abs()
  if gamma_on:
    _check(grads[:, 0, :c], dgr, dg_bound, what + " dgamma")
  # dx = a dy' + b x + c0 with a = gamma rs, b = -gamma rs^2 dgamma / n, c0 = -gamma rs dbeta / n - b mu: at most 8 fp32
  # roundings over the three terms, plus dgamma's own error carried by b into |x| + |mu|; then one output rounding
  rs, mu = srstd.to(F64).reshape(groups, 1, c), smean.to(F64).reshape(groups, 1, c)
  b = -gm * rs * rs * dgr[:, None] / n
  c0 = -gm * rs * dbr[:, None] / n - b * mu
  xg = x.to(F64).reshape(groups, rpg, c)
  terms = (gm * rs * gr.reshape(groups, rpg, c)).abs() + (b * xg).abs() + c0.abs()
  carried = (gm * rs * rs / n) * (xg.abs() + mu.abs()) * dg_bound[:, None]
  _check(dx.reshape(rows, c), dxr, _ulp(dxr, dtype) + (8 * U24 * terms + carried).reshape(rows, c), what + " dx", rpg)
  if dmask is not None:
    _exact(dmask.reshape(rows, c), gr, what + " masked dy", rpg)
  return path, bpath


@gpu
@pytest.mark.parametrize("c", [8, 24, 40, 64, 2048, 2728, 2736])
@pytest.mark.parametrize("dtype,fused", [(BF16, True), (BF16, False), (FP32, False)], ids=["bf16-fused", "bf16-pair", "fp32-pair"])
def test_bn_channels(record, c, dtype, fused):
  """Channel counts with idle threads (512 not a multiple of C / 8), the largest C the single-launch scratch holds (2728) and the
  first one above it; relu / residual / gamma / masked combinations alternate with C."""
  rows = 4096
  k = [8, 24, 40, 64, 2048, 2728, 2736].index(c)
  tags = ()
  if c == 2728:
    tags = (("C<=2728", "in"),)
  if c == 2736:
    tags = (("C<=2728", "out"),)
  run_bn_case(record, rows, c, 1, dtype, fused, relu=k % 2 == 0, residual=k % 3 == 1, gamma_on=k != 3, masked=k % 2 == 0, seed=10 + k, tags=tags)


@gpu
@pytest.mark.parametrize("relu,residual,gamma_on,masked", [(True, False, True, False), (False, False, True, False), (True, True, True, True), (False, True, False, False),
                                                           (True, False, False, True)])
@pytest.mark.parametrize("dtype,fused", [(BF16, True), (BF16, False), (FP32, False)], ids=["bf16-fused", "bf16-pair", "fp32-pair"])
def test_bn_flags(record, relu, residual, gamma_on, masked, dtype, fused):
  """relu / residual / gamma / masked backward on a ResNet-like tile (8 workers of 4 x 28 x 28 pixels, C = 64), per-worker groups."""
  run_bn_case(record, 8 * 3136, 64, 8, dtype, fused, relu, residual, gamma_on, masked, seed=30)


@gpu
@pytest.mark.parametrize("groups", ["1", "2", "3", "7", "sms", "sms+1"])
def test_bn_groups(record, groups):
  """Per-worker groups up to the SM count (one CTA per group at the cap) and one above it (the pair takes over)."""
  sms = _sms()
  g = {"sms": sms, "sms+1": sms + 1}.get(groups) or int(groups)
  c = 16
  rows = g * max(64, -(-4096 // g))
  plan = fused_plan(rows, c, g, False, False, sms)
  assert (plan is None) == (g > sms)
  tag = (("groups<=SMs", "in" if g <= sms else "out"),) if g >= sms else ()
  run_bn_case(record, rows, c, g, BF16, True, relu=True, residual=g == 3, masked=True, seed=40 + g, tags=tag)
  run_bn_case(record, rows, c, g, FP32, False, relu=g % 2 == 1, seed=50 + g)


@gpu
@pytest.mark.parametrize("c,groups,inside", [(2048, 8, True), (2064, 8, False), (64, 2, True)])
def test_bn_pairs_cap_and_replicas(record, c, groups, inside):
  """C * groups = 16384 (the workspace half is full: one replica) and 16512 (pair); C = 64 x 2 groups spreads over 8 replicas."""
  sms = _sms()
  rows = groups * (4096 if c == 64 else 512)
  limits = (72, 40, 1024)
  plan = fused_plan(rows, c, groups, False, False, sms, limits)
  assert (plan is not None) == inside
  if plan is not None:
    assert plan["replicas"] == (1 if c * groups == 16384 else 8), plan
    COVERAGE.add(("replicas", plan["replicas"]))
  tag = (("C*groups<=16384", "in" if inside else "out"),) if c * groups >= 16384 else ()
  run_bn_case(record, rows, c, groups, BF16, True, relu=True, residual=False, masked=True, seed=60 + c, limits=limits, tags=tag)


@gpu
@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("side", ["at", "below"])
def test_bn_min_rows(record, residual, side):
  """The fewest rows the single-launch kernel takes (4096, or 1024 with a fused residual / masked gradient) and one row fewer.
  C = 8 so that every row count is a legal tensor."""
  limit = DEFAULT_LIMITS[2] // 4 if residual else DEFAULT_LIMITS[2]
  rows = limit if side == "at" else limit - 1
  sms = _sms()
  for bwd in (False, True):
    assert (fused_plan(rows, 8, 1, bwd, residual, sms) is not None) == (side == "at")
  want = "fused" if side == "at" else "pair"
  run_bn_case(record, rows, 8, 1, BF16, True, relu=True, residual=residual, masked=residual, seed=70, expect=(want, want),
              tags=(("min_rows" + ("/4" if residual else ""), "in" if side == "at" else "out"),))


@gpu
@pytest.mark.parametrize("side", ["at", "above"])
def test_bn_size_caps(record, side):
  """The 72 MB forward / 40 MB backward caps, shrunk to 1 MB / 1 MB so the tensors stay small: exactly at the cap (fused) and one
  row above (pair). The forward and backward caps are crossed separately with a 2 MB forward cap."""
  c = 64
  at_rows = (1 << 20) // (2 * c)
  rows = at_rows if side == "at" else at_rows + 1
  sms = _sms()
  limits = (1, 1, 1024)
  assert (fused_plan(rows, c, 1, False, False, sms, limits) is not None) == (side == "at")
  assert (fused_plan(rows, c, 1, True, False, sms, limits) is not None) == (side == "at")
  want = "fused" if side == "at" else "pair"
  io = "in" if side == "at" else "out"
  run_bn_case(record, rows, c, 1, BF16, True, relu=True, seed=80, limits=limits, expect=(want, want), tags=(("max_mb_fwd", io), ("max_mb_bwd", io)))
  # forward inside a 2 MB cap while the backward is above its 1 MB cap
  run_bn_case(record, at_rows + 8, c, 1, BF16, True, relu=False, seed=81, limits=(2, 1, 1024), expect=("fused", "pair"))


def _rows_for(c, groups, bwd, target_vecs, sms):
  """Rows per group giving every CTA exactly `target_vecs` vectors (all CTAs at the per-group cap)."""
  octets = c // 8
  assert target_vecs % octets == 0
  cap = sms // groups
  return cap * (target_vecs // octets) * groups


@gpu
@pytest.mark.parametrize("bwd", [False, True], ids=["fwd", "bwd"])
@pytest.mark.parametrize("offset", [-1, 0, 1])
@pytest.mark.parametrize("residual", [False, True])
def test_bn_stash_boundary(record, bwd, offset, residual):
  """Per-CTA vectors one row below, at and one row above the on-chip stash (forward 11520, backward 5760 vectors): the re-read tail
  starts exactly at the boundary, for the residual loop and the plain loop."""
  sms = _sms()
  c, octets = 64, 8
  stash = STASH_BYTES // 16 // (2 if bwd else 1)
  rows = _rows_for(c, 1, bwd, stash + offset * octets, sms)
  plan = fused_plan(rows, c, 1, bwd, residual, sms)
  assert plan is not None and plan["ctas_per_group"] == sms
  assert plan["rows_per_cta"] * octets - plan["stash_vecs"] == offset * octets, plan
  side = {-1: "below", 0: "at", 1: "above"}[offset]
  COVERAGE.add(("stash", "bwd" if bwd else "fwd", side))
  run_bn_case(record, rows, c, 1, BF16, True, relu=True, residual=residual, masked=residual, seed=90 + offset)


@gpu
def test_bn_uneven_and_empty_chunks(record):
  """Rows per group that the CTAs do not divide evenly, down to chunks that hold no row at all (nvec == 0)."""
  sms = _sms()
  c = 512
  rows = None
  for r in range(4096, 20000, 2):
    plan = fused_plan(r, c, 1, False, False, sms)
    if plan is not None and plan["empty_chunks"] > 0 and fused_plan(r, c, 1, True, False, sms)["empty_chunks"] > 0:
      rows = r
      break
  assert rows is not None
  COVERAGE.add(("empty_chunks",))
  run_bn_case(record, rows, c, 1, BF16, True, relu=True, residual=True, masked=True, seed=100)
  # two groups whose rows the CTAs do not divide evenly
  for r in range(4096 * 2, 40000, 2):
    plan = fused_plan(r, 64, 2, False, False, sms)
    if plan is not None and (r // 2) % plan["ctas_per_group"]:
      run_bn_case(record, r, 64, 2, BF16, True, relu=False, seed=101)
      break


@gpu
def test_bn_sequences(record):
  """Back-to-back single-launch calls of different C * groups (each must find its workspace half zeroed), then pair calls after a
  single-launch call with a larger C * groups, then pair calls whose ticket word moves (it sits after the C * groups sums)."""
  for c, groups, rows in ((2048, 8, 8 * 512), (64, 1, 8192), (512, 4, 4 * 1024), (2048, 8, 8 * 512), (24, 3, 3 * 2048)):
    assert run_bn_case(record, rows, c, groups, BF16, True, relu=True, seed=110 + c, limits=(72, 40, 1024)) == ("fused", "fused")
  for c, groups, rows in ((512, 4, 4 * 256), (2048, 8, 8 * 128), (64, 1, 512), (1024, 4, 4 * 128)):
    run_bn_case(record, rows, c, groups, BF16, False, relu=True, seed=120 + c)
    run_bn_case(record, rows, c, groups, FP32, True, relu=False, seed=130 + c)


@gpu
def test_bn_cuda_graph_replay(record):
  """Three single-launch forwards captured in one CUDA graph (an odd count: the device-side workspace toggle ends on the other half),
  replayed twice; both replays match the oracle."""
  from aggregathor_b200.ops import nn_native
  cases = [(8192, 64, 1), (4 * 2048, 256, 4), (8 * 512, 2048, 8)]
  ops_in = []
  for k, (rows, c, groups) in enumerate(cases):
    x, gamma, beta = _bn_operands(rows, c, groups, BF16, 140 + k)
    mm0, mv0 = _grid((c,), -2, 2, 150 + k, FP32), _grid((c,), 1, 4, 160 + k, FP32)
    ops_in.append((x, gamma, beta, mm0, mv0, mm0.clone(), mv0.clone(), groups))
  for x, gamma, beta, mm0, mv0, mm, mv, groups in ops_in:   # warm-up: workspaces and kernel attributes before capture
    nn_native.batchnorm_forward(_as_nhwc(x), gamma, beta, mm.clone(), mv.clone(), DECAY, EPS, True, groups)
  torch.cuda.synchronize()
  graph = torch.cuda.CUDAGraph()
  stream = torch.cuda.Stream()
  stream.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(stream):
    with torch.cuda.graph(graph, stream=stream):
      outs = [nn_native.batchnorm_forward(_as_nhwc(x), gamma, beta, mm, mv, DECAY, EPS, True, groups) for x, gamma, beta, mm0, mv0, mm, mv, groups in ops_in]
  torch.cuda.current_stream().wait_stream(stream)
  assert all(s == 0 for n, s in record.calls if n == "agb_bn_forward_fused")
  for replay in range(2):
    for x, gamma, beta, mm0, mv0, mm, mv, groups in ops_in:
      mm.copy_(mm0)
      mv.copy_(mv0)
    graph.replay()
    torch.cuda.synchronize()
    for (x, gamma, beta, mm0, mv0, mm, mv, groups), (y, mean, rstd) in zip(ops_in, outs):
      yr, mr, rr, mmr, mvr = bn_forward_ref(x, gamma, beta, mm0, mv0, DECAY, EPS, True, groups)
      what = "graph replay %d C=%d groups=%d" % (replay, x.shape[1], groups)
      rpg = x.shape[0] // groups
      _exact(mean, mr.to(FP32), what + " save_mean")
      _check(rstd, rr, 2.0 ** -21 * rr, what + " save_rstd")
      scale = (rr.reshape(groups, -1) * gamma.to(F64)).repeat_interleave(rpg, dim=0)
      shift = beta.to(F64).abs() + (mr.reshape(groups, -1) * rr.reshape(groups, -1) * gamma.to(F64)).abs().repeat_interleave(rpg, dim=0)
      _check(y.reshape(x.shape), yr, _y_bound(x, scale, shift, None, yr, BF16, 2.0 ** -21), what + " y", rpg)
      _check(mm, mmr, 4 * U24 * (DECAY * mm0.to(F64).abs() + (1 - DECAY) * mr[:x.shape[1]].abs()) + 1e-300, what + " moving_mean")
  COVERAGE.add(("graph",))


@gpu
@pytest.mark.parametrize("dtype,ratio", [(BF16, 0), (BF16, 8), (BF16, 64), (FP32, 0), (FP32, 100), (FP32, 1000)])
@pytest.mark.parametrize("step", ["first", "later"])
@pytest.mark.parametrize("fused", [True, False], ids=["fused", "pair"])
def test_bn_variance_conditioning(record, dtype, ratio, step, fused):
  """Random operands with |mean| / std = ratio, with a zero moving mean (first step) and with the moving mean at the batch mean
  (later steps). C = 64, 32 x 28 x 28 rows (25088)."""
  from aggregathor_b200.ops import nn_native
  if dtype == FP32 and fused:
    pytest.skip("fp32 activations only run on the statistics + apply pair")
  nn_native.set_bn_fused(fused)
  rows, c = 25088, 64
  gen = torch.Generator(device="cuda").manual_seed(170 + ratio)
  signs = torch.where(torch.arange(c, device="cuda") % 2 == 0, 1.0, -1.0)
  x = (torch.randn((rows, c), device="cuda", generator=gen, dtype=F64) + ratio * signs).to(dtype)
  gamma, beta = torch.ones(c, device="cuda"), torch.zeros(c, device="cuda")
  yr, mr, rr, _, _ = bn_forward_ref(x, gamma, beta, torch.zeros(c, device="cuda"), torch.ones(c, device="cuda"), DECAY, EPS, False, 1)
  mm = torch.zeros(c, device="cuda") if step == "first" else mr.to(FP32)
  mv = torch.ones(c, device="cuda")
  y, mean, rstd, path = _bn_forward(record, x, gamma, beta, mm, mv, False, 1, None)
  assert path == ("fused" if fused else "pair")
  what = "bn conditioning %s %s |mean|/std=%d %s step" % (path, dtype, ratio, step)
  # With a pivot p per channel, the kernels sum d = x - p and d^2 in fp32 chains of L <= rows per thread + lanes additions
  # (about 50 + 64 here); the variance is E[d^2] - E[d]^2 evaluated in fp64 from those sums, so its relative error is at most
  # L u (1 + (mean - p)^2 / var). A pivot within a few std of the mean (a sample of the batch, or the moving mean at the batch mean)
  # keeps the factor below ~20: 2 L u * 20 ~ 3e-4 worst case, ~1e-6 expected for sums of random-signed rounding errors; rstd
  # inherits half of it plus the 5 u of `save_rstd` above. Without a pivot the factor is ratio^2 + 1 (1e6 at ratio 1000).
  # The assert takes 1e-5. The saved mean has the same 1e-5 std from the sums, plus its own rounding to fp32: half an ulp of
  # |mean| (3e-5 at |mean| = 1000).
  _check(rstd, rr, 1e-5 * rr, what + " save_rstd")
  _check(mean, mr, 1e-5 / rr + 0.5 * _ulp(mr, FP32), what + " save_mean")


@gpu
def test_bn_nonfinite(record):
  """NaN and +-inf planted in one channel of one group of x, and a NaN in the residual: exactly the oracle's non-finite outputs are
  non-finite (NaN survives the ReLU), every other element meets the bound; single-launch, bf16 pair and fp32 pair."""
  from aggregathor_b200.ops import nn_native
  rows, c, groups = 4 * 2048, 64, 4
  rpg = rows // groups
  for dtype, fused in ((BF16, True), (BF16, False), (FP32, False)):
    for residual in (False, True):
      nn_native.set_bn_fused(fused)
      x, gamma, beta = _bn_operands(rows, c, groups, dtype, 180)
      x[rpg + 5, 3] = float("nan")
      x[2 * rpg + 7, 9] = float("inf")
      x[3 * rpg + 1, 17] = float("-inf")
      res = _grid((rows, c), -3, 3, 181, dtype) if residual else None
      if residual:
        res[11, 20] = float("nan")
        res[12, 21] = float("inf")
      mm, mv = torch.zeros(c, device="cuda"), torch.ones(c, device="cuda")
      y, mean, rstd, path = _bn_forward(record, x, gamma, beta, mm, mv, True, groups, res)
      assert path == ("fused" if fused else "pair")
      yr, mr, rr, _, _ = bn_forward_ref(x, gamma, beta, torch.zeros(c, device="cuda"), torch.ones(c, device="cuda"), DECAY, EPS, True, groups, res)
      scale = (rr.reshape(groups, c) * gamma.to(F64)).repeat_interleave(rpg, dim=0)
      shift = beta.to(F64).abs() + (mr.reshape(groups, c) * rr.reshape(groups, c) * gamma.to(F64)).abs().repeat_interleave(rpg, dim=0)
      bound = _y_bound(x.masked_fill(~torch.isfinite(x), 0), scale.nan_to_num(), shift.nan_to_num(), res.masked_fill(~torch.isfinite(res), 0) if residual else None, yr.nan_to_num(), dtype, 2.0 ** -21)
      _check(y, yr, bound, "bn nonfinite %s %s residual=%d y" % (path, dtype, residual), rpg)
      COVERAGE.add(("nonfinite", path, str(dtype)))


@gpu
def test_bn_coverage():
  """Runs last: the batch-norm cases above went through every implementation and both sides of every envelope boundary."""
  if not any(k[0] == "forward" for k in COVERAGE):
    pytest.skip("needs the batch-norm tests of this module in the same run")
  want = [("forward", "fused", str(BF16)), ("backward", "fused", str(BF16)), ("forward", "pair", str(BF16)), ("backward", "pair", str(BF16)),
          ("forward", "pair", str(FP32)), ("backward", "pair", str(FP32)), ("graph",), ("empty_chunks",), ("replicas", 1), ("replicas", 8)]
  for bound in ("min_rows", "min_rows/4", "max_mb_fwd", "max_mb_bwd", "C<=2728", "groups<=SMs", "C*groups<=16384"):
    want.append(("forward", "fused", bound, "in"))
    want.append(("forward", "pair", bound, "out"))
  for direction in ("fwd", "bwd"):
    for side in ("below", "at", "above"):
      want.append(("stash", direction, side))
  missing = [w for w in want if w not in COVERAGE]
  assert not missing, missing


# ---------------------------------------------------------------------------- #
# Column sums

@gpu
@pytest.mark.parametrize("dtype", [BF16, FP32])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("groups", [1, 3])
def test_colsum(dtype, masked, groups):
  """Bias gradients: per-group column sums written `group_stride` apart; grid operands make them exact in any order."""
  from aggregathor_b200.ops import nn_native
  for rows, c in ((groups * 4096, 64), (groups * 333, 2056), (groups * 1, 8)):
    dy = _grid((rows, c), -8, 8, 190 + c, dtype)
    y = _grid((rows, c), -2, 2, 191 + c, dtype) if masked else None
    if y is not None:
      y[0, 0] = float("nan")
    stride = c + 16
    buf = torch.full((groups, stride), -7.0, dtype=FP32, device="cuda")
    nn_native.colsum(dy, y, out=buf[0, :c], groups=groups, group_stride=stride)
    _exact(buf[:, :c], colsum_ref(dy, y, groups), "colsum %s masked=%d groups=%d C=%d" % (dtype, masked, groups, c))
    assert bool((buf[:, c:] == -7.0).all())


# ---------------------------------------------------------------------------- #
# LayerNorm

@gpu
@pytest.mark.parametrize("rows", [1, 7, 333, 50000])
@pytest.mark.parametrize("c", [8, 264, 1024, 5632])
def test_layernorm(rows, c):
  from aggregathor_b200.ops import nn_native
  if rows * c > 50000 * 1024:
    rows = 50000 * 1024 // c
  x = _grid((rows, c), -8, 8, 200 + c, BF16)
  gamma, beta = _grid((c,), 2, 6, 201, FP32) / 4, _grid((c,), -4, 4, 202, FP32) / 8
  y, mean, rstd = nn_native.layernorm_forward(x, gamma, beta, EPS)
  yr, mr, rr = layernorm_forward_ref(x, gamma, beta, EPS)
  what = "layernorm rows=%d C=%d" % (rows, c)
  # the lanes sum d = x - p (p: the row's first element) and d^2: integers, exact. mean = p + sum / C: two roundings, u |mean - p|
  # and one half ulp of the mean
  m = (mr - x[:, 0].to(F64)).abs()
  dmean = _ulp(mr, FP32) + 2 * U24 * m
  _check(mean, mr, dmean, what + " mean")
  # var = sumsq / C - (sum / C)^2: four roundings on sumsq / C = var + m^2 and m^2, i.e. a relative error of u (3 + 4 m^2 / var)
  # on var (eps add included); the square root halves it, rsqrtf adds 2 ulp (<= 2^-22)
  vr = 1.0 / rr ** 2 - EPS
  rel = 0.5 * U24 * (3 + 4 * m ** 2 / vr.clamp_min(EPS)) + 2.0 ** -22
  _check(rstd, rr, rel * rr, what + " rstd")
  # y = (x - mean) * rstd * gamma + beta: the mean's error times rstd gamma, the rstd error, 4 fp32 roundings on the terms, then
  # one output rounding
  terms = ((x.to(F64) - mr[:, None]) * rr[:, None] * gamma.to(F64)).abs()
  bound = _ulp(yr, BF16) + (rel[:, None] + 4 * U24) * terms + (dmean * rr)[:, None] * gamma.to(F64) + 2 * U24 * (terms + beta.to(F64).abs())
  _check(y, yr, bound, what + " y")
  dy = _grid((rows, c), -4, 4, 203 + c, BF16)
  gg, gb = torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
  dx = nn_native.layernorm_backward(dy, x, gamma, mean, rstd, gg, gb)
  dxr, dgr, dbr = layernorm_backward_ref(dy, x, gamma, mean, rstd)
  # dbeta: sums of integers (exact); dgamma: terms dy * xhat with 3 roundings each, summed in shared-memory fp32 atomics over a
  # CTA's rows, then fp32 atomics over the (<= 4 x SM count) CTAs: |err| <= (rows + 4 SMs + 3) u * sum|dy xhat|
  _exact(gb, dbr, what + " dbeta")
  xhat = (x.to(F64) - mean.to(F64)[:, None]) * rstd.to(F64)[:, None]
  _check(gg, dgr, (rows + 4 * _sms() + 3) * U24 * (dy.to(F64) * xhat).abs().sum(dim=0), what + " dgamma")
  # dx = rs (g - s1 - xhat s2): s1, s2 are means of warp sums of C terms (chains of C / 32 + 5 additions after up to 4 roundings
  # per term, one division); then up to 7 roundings over |g| + |s1| + |xhat s2|, and the output rounding
  g = dy.to(F64) * gamma.to(F64)
  chain = c // 32 + 10
  s1e = chain * U24 * g.abs().mean(dim=1, keepdim=True)
  s2e = chain * U24 * (g * xhat).abs().mean(dim=1, keepdim=True)
  r = rstd.to(F64)[:, None]
  terms = g.abs() + g.mean(dim=1, keepdim=True).abs() + (xhat * (g * xhat).mean(dim=1, keepdim=True)).abs()
  _check(dx, dxr, _ulp(dxr, BF16) + r * (s1e + xhat.abs() * s2e) + 8 * U24 * r * terms, what + " dx")


@gpu
def test_layernorm_wide_rows_and_conditioning():
  """C = 5640 is above the native kernels (the aten provider serves it); a row of mean 64 and std 1 over C = 4096 keeps its
  variance (rstd within 1e-5, see `test_bn_variance_conditioning` for the derivation with a sample pivot)."""
  from aggregathor_b200.ops import nn_native
  x = _grid((4, 5640), -8, 8, 210, BF16)
  assert nn_native.layernorm_forward(x, torch.ones(5640, device="cuda"), torch.zeros(5640, device="cuda"), EPS) is None
  gen = torch.Generator(device="cuda").manual_seed(211)
  c = 4096
  x = (torch.randn((333, c), device="cuda", generator=gen) + 64).to(BF16)
  _, mean, rstd = nn_native.layernorm_forward(x, torch.ones(c, device="cuda"), torch.zeros(c, device="cuda"), EPS)
  _, mr, rr = layernorm_forward_ref(x, torch.ones(c, device="cuda"), torch.zeros(c, device="cuda"), EPS)
  _check(rstd, rr, 1e-5 * rr, "layernorm mean 64 std 1 rstd")


# ---------------------------------------------------------------------------- #
# Softmax cross-entropy

def _xent_bounds(logits, t, logp, n, dtype):
  """Per-row bounds for rows of finite logits, `n` rows per group. __expf(x) is within 2 + 1.16 |x| ulp and __logf within
  2^-21.41 absolute on [0.5, 2], 3 ulp elsewhere (CUDA math accuracy tables).
  sum = sum exp(z - mx) >= 1: each term carries the rounding of z - mx (u |x| relative after exp) and the expf error, and the
  lanes' fp32 chains of K / 32 + 5 additions add (K / 32 + 5) u: relative error e_s;
  lse = mx + log(sum): |err| <= e_s + log error + u |lse|; logp = z - lse: + u |logp|;
  p = exp(logp) turns the logp error into a relative one and adds its own expf error; (p - t) * (1 / n): three more roundings
  (the subtraction, 1 / n, the product), then the output rounding.
  The loss of a row is -sum t logp (one rounding per product, chains of K / 32 + 6), then fp32 atomics of (row * (1 / n)).
  Returns (dlogits bound [rows, K], loss error [rows], |row loss| [rows])."""
  k = logits.shape[1]
  z = logits.to(F64)
  mx = z.max(dim=1, keepdim=True).values
  lse = (z - logp)[:, :1]
  x = (z - mx).abs()
  e = torch.exp(-x)
  e_s = (e * (2 + 1.16 * x + 0.5 * x) * 2 * U24).sum(dim=1, keepdim=True) / e.sum(dim=1, keepdim=True) + (k / 32 + 5) * U24
  log_sum = (lse - mx).abs()
  e_log = torch.where(log_sum <= math.log(2), torch.full_like(log_sum, 2 ** -21.41), 6 * U24 * log_sum)
  e_logp = e_s + e_log + U24 * lse.abs() + U24 * logp.abs()
  p = torch.exp(logp)
  e_p = p * (e_logp * 1.01 + (2 + 1.16 * logp.abs()) * 2 * U24)
  ref_d = (p - t) / n
  d_bound = (e_p + 3 * U24 * (p - t).abs()) / n + _ulp(ref_d, dtype)
  row = -(t * logp).sum(dim=1)
  row_err = (t * e_logp).sum(dim=1) + (k / 32 + 7) * U24 * (t * logp).abs().sum(dim=1)
  return d_bound, row_err, row.abs()


@gpu
@pytest.mark.parametrize("k", [10, 31, 32, 33, 1000, 1001, 21843])
@pytest.mark.parametrize("groups", [1, 4])
@pytest.mark.parametrize("smoothing", [0.0, 0.1])
@pytest.mark.parametrize("dtype", [BF16, FP32])
def test_softmax_xent(k, groups, smoothing, dtype):
  """Labels at 0 and K - 1, rows spread over +-80, rows of equal logits, strided logits whose padding columns of dlogits keep a
  sentinel, and a NaN logit that poisons its own row only."""
  from aggregathor_b200.ops import nn_native
  b = 16
  ld = k + 8 - k % 8 + 8
  gen = torch.Generator(device="cpu").manual_seed(220 + k)
  base = torch.full((b, ld), 5.0, dtype=F64)
  base[:, :k] = (torch.rand((b, k), generator=gen, dtype=F64) * 160 - 80)
  base[1, :k] = 3.0                                              # all logits equal
  base[2, :k] = (torch.rand(k, generator=gen, dtype=F64) * 4 - 2)
  logits = base.to(dtype).cuda()[:, :k]
  labels = torch.randint(0, k, (b,), generator=gen)
  labels[0], labels[1], labels[2] = 0, k - 1, k - 1
  labels = labels.cuda()
  nan_row = 5
  logits[nan_row, k // 2] = float("nan")
  dl_buf = torch.full((b, ld), 77.0, dtype=dtype, device="cuda")
  from aggregathor_b200.ops.nn_native import _fn, _ptr, _stream, _check as _status
  import ctypes
  loss = torch.empty((groups,), dtype=FP32, device="cuda")
  _status(_fn("agb_softmax_xent", logits)(_ptr(logits), _ptr(labels), _ptr(dl_buf), _ptr(loss), ctypes.c_int(b), ctypes.c_int(k), ctypes.c_longlong(ld),
                                            ctypes.c_float(smoothing), ctypes.c_int(groups), _stream()), "softmax_xent")
  assert bool((dl_buf[:, k:] == 77.0).all()), "dlogits written past K"
  lr, dr, t, logp = softmax_xent_ref(logits, labels, float(torch.tensor(smoothing, dtype=FP32)), groups)
  what = "xent K=%d groups=%d smoothing=%g %s" % (k, groups, smoothing, dtype)
  n = b // groups
  finite = torch.arange(b, device="cuda") != nan_row
  d_bound, row_err, row_abs = _xent_bounds(logits[finite], t[finite], logp[finite], n, dtype)
  full = torch.zeros((b, k), dtype=F64, device="cuda")
  full[finite] = d_bound
  _check(dl_buf[:, :k], dr, full, what + " dlogits")
  err, mag = torch.zeros(b, dtype=F64, device="cuda"), torch.zeros(b, dtype=F64, device="cuda")
  err[finite], mag[finite] = row_err, row_abs
  _check(loss, lr, (err.reshape(groups, n).sum(dim=1) + (n + 2) * U24 * mag.reshape(groups, n).sum(dim=1)) / n, what + " loss")


# ---------------------------------------------------------------------------- #
# Pools, ReLU, image normalisation

@gpu
@pytest.mark.parametrize("k,s", [(2, 2), (3, 2), (3, 1), (5, 2)])
@pytest.mark.parametrize("dtype", [BF16, FP32])
def test_maxpool(k, s, dtype):
  """Grid inputs in [-2, 2] (ties everywhere): values and window-relative argmax bit-exact, every padding parity, NaN windows;
  the backward with integer dy exact (3 x 3 / 2 takes its 2 x 2-block kernel, the others the generic gather)."""
  from aggregathor_b200.ops import nn_native
  for h, w in ((9, 8), (10, 11)):
    for pads in ((0, 0, 0, 0), (1, 1, 1, 1), (0, 1, 1, 0), (1, 0, 0, 1), (k // 2, k - 1 - k // 2, k - 1 - k // 2, k // 2)):
      x = _grid((3, 16, h, w), -2, 2, 230 + h + k, dtype).contiguous(memory_format=CL)
      x[0, 3, 4, 4] = float("nan")
      x[1, 8, 0, 0] = float("nan")
      x[2, 9, 2, 3] = float("inf")
      x[2, 10, 5, 5] = float("-inf")
      y, arg = nn_native.maxpool_forward(x, k, s, pads)
      vr, ir = maxpool_forward_ref(x, k, s, pads)
      what = "maxpool k=%d s=%d pads=%s %s %dx%d" % (k, s, pads, dtype, h, w)
      _exact(y, vr, what + " values")
      got = arg.permute(0, 3, 1, 2).long()
      if not torch.equal(got, ir):
        first = (got != ir).nonzero()[0].tolist()
        raise AssertionError("%s argmax: first difference at %s: %d vs oracle %d" % (what, first, int(got[tuple(first)]), int(ir[tuple(first)])))
      dy = _grid(tuple(y.shape), -4, 4, 240 + k, dtype).contiguous(memory_format=CL)
      dx = nn_native.maxpool_backward(dy, x.shape, arg, k, s, pads)
      _exact(dx, maxpool_backward_ref(dy, ir, x.shape, k, s, pads), what + " backward")


@gpu
def test_maxpool_tall_maps():
  """Maps tall enough that the backward launches in several slices of images (grid.y = images x rows <= 65535)."""
  from aggregathor_b200.ops import nn_native
  for k, s, pads in ((3, 2, (1, 1, 1, 1)), (2, 2, (0, 0, 0, 0))):
    x = _grid((40, 8, 4000, 8), -2, 2, 250 + k, BF16).contiguous(memory_format=CL)
    y, arg = nn_native.maxpool_forward(x, k, s, pads)
    vr, ir = maxpool_forward_ref(x, k, s, pads)
    _exact(y, vr, "tall maxpool k=%d values" % k)
    assert torch.equal(arg.permute(0, 3, 1, 2).long(), ir)
    dy = _grid(tuple(y.shape), -4, 4, 251, BF16).contiguous(memory_format=CL)
    _exact(nn_native.maxpool_backward(dy, x.shape, arg, k, s, pads), maxpool_backward_ref(dy, ir, x.shape, k, s, pads), "tall maxpool k=%d backward" % k)


@gpu
@pytest.mark.parametrize("dtype", [BF16, FP32])
def test_global_avgpool(dtype):
  """Mean over H x W: the fp32 sum of HW terms in one chain (HW u relative to sum|x|), a product by the rounded 1 / HW (2 u), the
  output rounding (one ulp). Backward: dy * (1 / HW) rounded twice, then the output rounding."""
  from aggregathor_b200.ops import nn_native
  gen = torch.Generator(device="cuda").manual_seed(260)
  for n, c, h, w in ((5, 64, 7, 7), (3, 2056, 1, 1), (2, 8, 17, 13)):
    x = (torch.randn((n, c, h, w), device="cuda", generator=gen) * 3).to(dtype).contiguous(memory_format=CL)
    y = nn_native.global_avgpool_forward(x)
    ref = avgpool_ref(x)
    hw = h * w
    _check(y.reshape(n, c), ref, _ulp(ref, dtype) + (hw + 2) * U24 * x.to(F64).abs().mean(dim=(2, 3)), "avgpool %s %s" % (dtype, (n, c, h, w)))
    dy = (torch.randn((n, c, 1, 1), device="cuda", generator=gen)).to(dtype)
    dx = nn_native.global_avgpool_backward(dy, (n, c, h, w))
    dref = (dy.to(F64) / hw).expand(n, c, h, w)
    _check(dx, dref, _ulp(dref, dtype) + 2 * U24 * dref.abs(), "avgpool backward %s" % dtype)


@gpu
@pytest.mark.parametrize("mode", ["vgg", "inception", "lenet"])
@pytest.mark.parametrize("dtype", [BF16, FP32])
def test_image_normalize(mode, dtype):
  """(x - mean[c]) * scale: the mean and scale rounded to fp32 (u each, relative to 255 and |ref|), the difference and the product
  (2 u), the output rounding (one ulp)."""
  from aggregathor_b200.ops import nn_native
  images = _grid((3, 17, 19, 3), 0, 255, 270, torch.uint8)
  out = nn_native.image_normalize(images, mode, dtype)
  ref = image_normalize_ref(images, mode)
  _, scale = IMAGE_MODES[mode]
  _check(out.permute(0, 2, 3, 1), ref, _ulp(ref, dtype) + 4 * U24 * (ref.abs() + 256 * scale), "image_normalize %s %s" % (mode, dtype))


@gpu
@pytest.mark.parametrize("dtype", [BF16, FP32])
def test_nonfinite_relu_add_relu6_softmax(dtype):
  """NaN and +-inf at known positions: ReLU and add + ReLU keep NaN and +inf, map -inf to 0; ReLU6 keeps NaN; softmax cross-entropy
  poisons exactly the row of a NaN logit."""
  from aggregathor_b200.ops import nn_native
  a = _grid((64, 24), -3, 3, 280, dtype)
  b = _grid((64, 24), -3, 3, 281, dtype)
  a[1, 2], a[3, 4], a[5, 6], b[7, 8], b[9, 10] = float("nan"), float("inf"), float("-inf"), float("nan"), float("-inf")
  for other in (None, b):
    out = nn_native.add_relu_forward(a, other if other is not None else torch.zeros_like(a), True)
    s = a.to(F64) + (other.to(F64) if other is not None else 0)
    ref = torch.where(s > 0, s, torch.where(torch.isnan(s), s, torch.zeros_like(s)))
    _exact(out, ref, "add_relu %s residual=%d" % (dtype, other is not None))
  if dtype == BF16:
    x = _grid((64, 24), -8, 8, 282, BF16)
    x[0, 0], x[1, 1], x[2, 2] = float("nan"), float("inf"), float("-inf")
    out = nn_native.relu6(x)
    xf = x.to(F64)
    ref = torch.where(torch.isnan(xf), xf, xf.clamp(0, 6))
    _exact(out, ref, "relu6")
  logits = _grid((8, 40), -5, 5, 283, dtype)
  logits[3, 7] = float("nan")
  loss, dl = nn_native.softmax_xent(logits, torch.arange(8, device="cuda") % 40, 0.0, 2)
  assert torch.isnan(dl[3]).all() and torch.isfinite(dl[torch.arange(8, device="cuda") != 3]).all()
  assert torch.isnan(loss[0]) and torch.isfinite(loss[1])

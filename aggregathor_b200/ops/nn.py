"""Neural-network ops with two providers.

`backend == "native"`: hand-written sm_90a kernels from `native/op_nn` (wgmma/TMA GEMM and
implicit-GEMM convolution, fused BN/ReLU/residual, pooling, softmax-CE). `backend == "torch"`: aten
library calls — the fp32/bf16 numerical reference of every kernel test and the baseline arm.
A native op that is not available for a given shape falls back to the torch provider *only* when
`AGB_NATIVE_STRICT` is unset; with `AGB_NATIVE_STRICT=1` it raises, so a silent library fallback
cannot masquerade as the native path.

Tensor conventions: activations (N, C, H, W) with channels_last strides (NHWC memory); conv weights
are tensors of shape [Cout, kh, kw, Cin] (OHWI memory); linear weights [out, in].
"""

import math
import os

import torch
import torch.nn.functional as F

from .. import tools

_CL = torch.channels_last
_STRICT = bool(os.environ.get("AGB_NATIVE_STRICT", ""))


def _native():
  from . import nn_native
  return nn_native


fallbacks = {}   # op name -> number of times the torch provider served a call made with backend == "native" (diagnostics, tests)


def set_strict(flag):
  """Raise instead of falling back to the torch provider when a native op cannot take its arguments."""
  global _STRICT
  _STRICT = bool(flag)


def _fallback(op):
  fallbacks[op] = fallbacks.get(op, 0) + 1
  if _STRICT:
    raise tools.UserException("Native op " + repr(op) + " unavailable for these arguments and AGB_NATIVE_STRICT is set")


def _pad_input(x, pads, value=0.0):
  t, b, l, r = pads
  if t == b and l == r:
    return x, (t, l)
  return F.pad(x, (l, r, t, b), value=value), (0, 0)


def _relu_mask(dy, y):
  return dy * (y > 0).to(dy.dtype)


def group_view(tensor, group, stride):
  """View of the same shape `stride` * `group` elements further in the underlying buffer: the gradient of logical worker
  `group` when `tensor` is worker 0's view into the [w, d] gradient matrix."""
  if tensor is None or group == 0:
    return tensor
  return tensor.as_strided(tensor.shape, tensor.stride(), tensor.storage_offset() + group * stride)


def _chunks(tensor, groups):
  return tensor.chunk(groups, dim=0) if tensor is not None else [None] * groups


# ---------------------------------------------------------------------------- #
# Convolution

def conv2d_forward(backend, x, weight, bias, stride, pads, relu, aux=None):
  """`aux`: dict owned by the calling layer, handed back to `conv2d_backward` (provider-private forward by-products)."""
  if backend == "native" and x.is_cuda:
    out = _native().conv2d_forward(x, weight, bias, stride, pads, relu, aux)
    if out is not None:
      return out
    _fallback("conv2d_forward")
  xp, padding = _pad_input(x, pads)
  y = F.conv2d(xp, weight.permute(0, 3, 1, 2), bias.to(x.dtype) if bias is not None else None, stride=stride, padding=padding)
  if relu:
    y = torch.relu_(y)
  return y.contiguous(memory_format=_CL)


def conv2d_backward(backend, dy, x, weight, y, stride, pads, relu, has_bias, need_dx, grad_w, grad_b, groups=1, group_stride=0, aux=None, addend=None):
  """Writes dW into `grad_w` ([Cout, kh, kw, Cin] fp32 view) and db into `grad_b`; returns dx or None. With `groups` > 1 the batch
  is `groups` consecutive per-worker batches and worker g's gradients go `g * group_stride` elements after worker 0's.
  `addend` (x's shape, with `need_dx`): returns `add_forward(addend, dx)` instead of dx; the native 1x1 stride-1 data gradient sums it
  in its epilogue, every other case adds it separately."""
  if addend is not None:
    if backend == "native" and x.is_cuda:
      out = _native().conv2d_backward(dy, x, weight, y, stride, pads, relu, has_bias, need_dx, grad_w, grad_b, groups, group_stride, aux, addend)
      if out is not NotImplemented:
        return out, None, None
    dx, _, _ = conv2d_backward(backend, dy, x, weight, y, stride, pads, relu, has_bias, need_dx, grad_w, grad_b, groups, group_stride, aux)
    return add_forward(backend, addend, dx), None, None
  if backend == "native" and x.is_cuda:
    out = _native().conv2d_backward(dy, x, weight, y, stride, pads, relu, has_bias, need_dx, grad_w, grad_b, groups, group_stride, aux)
    if out is not NotImplemented:
      return out, None, None
    _fallback("conv2d_backward")
  if groups > 1:
    pieces = []
    for g, (dy_g, x_g, y_g) in enumerate(zip(_chunks(dy, groups), _chunks(x, groups), _chunks(y, groups))):
      dx_g, _, _ = conv2d_backward(backend, dy_g.contiguous(memory_format=_CL), x_g.contiguous(memory_format=_CL), weight, y_g, stride, pads, relu, has_bias, need_dx,
                                   group_view(grad_w, g, group_stride), group_view(grad_b, g, group_stride))
      pieces.append(dx_g)
    return (torch.cat(pieces, dim=0).contiguous(memory_format=_CL) if need_dx else None), None, None
  if relu:
    dy = _relu_mask(dy, y)
  t, b, l, r = pads
  xp, padding = _pad_input(x, pads)
  w = weight.permute(0, 3, 1, 2)
  dxp, dw, db = torch.ops.aten.convolution_backward(
    dy, xp, w, [weight.shape[0]] if has_bias else None, [stride, stride], list(padding), [1, 1], False, [0, 0], 1, [need_dx, True, has_bias])
  grad_w.copy_(dw.permute(0, 2, 3, 1))
  if has_bias:
    grad_b.copy_(db)
  dx = None
  if need_dx:
    dx = dxp if padding != (0, 0) or (t == 0 and b == 0 and l == 0 and r == 0) else dxp[:, :, t:dxp.shape[2] - b, l:dxp.shape[3] - r]
    dx = dx.contiguous(memory_format=_CL)
  return dx, None, None


# ---------------------------------------------------------------------------- #
# Depthwise convolution (weights [C * multiplier, k, k, 1]; `pads` = (top, bottom, left, right))

def depthwise_forward(backend, x, weight, stride, pads):
  if backend == "native" and x.is_cuda:
    out = _native().depthwise_forward(x, weight, stride, pads)
    if out is not None:
      return out
    _fallback("depthwise_forward")
  t, b, l, r = pads
  xp = F.pad(x, (l, r, t, b))
  return F.conv2d(xp, weight.permute(0, 3, 1, 2), None, stride, 0, 1, x.shape[1]).contiguous(memory_format=_CL)


def depthwise_backward(backend, dy, x, weight, stride, pads, grad_w, groups=1, group_stride=0):
  """Returns dx; the weight gradient of every logical worker goes into its row (`grad_w` = worker 0's [C * multiplier, k, k, 1] view)."""
  if backend == "native" and x.is_cuda:
    out = _native().depthwise_backward(dy, x, weight, stride, pads, grad_w, groups, group_stride)
    if out is not None:
      return out
    _fallback("depthwise_backward")
  t, b, l, r = pads
  n, c, h, w = x.shape
  xp = F.pad(x, (l, r, t, b))
  kernel = weight.permute(0, 3, 1, 2)
  pieces = []
  for g, (dy_g, xp_g) in enumerate(zip(_chunks(dy, groups), _chunks(xp, groups))):
    dxp, dw, _ = torch.ops.aten.convolution_backward(dy_g, xp_g, kernel, None, [stride, stride], [0, 0], [1, 1], False, [0, 0], c, [True, True, False])
    group_view(grad_w, g, group_stride).copy_(dw.permute(0, 2, 3, 1))
    pieces.append(dxp)
  dxp = pieces[0] if len(pieces) == 1 else torch.cat(pieces, dim=0)
  return dxp[:, :, t:t + h, l:l + w].contiguous(memory_format=_CL)


# ---------------------------------------------------------------------------- #
# Dense

def linear_forward(backend, x, weight, bias, relu):
  if backend == "native" and x.is_cuda:
    out = _native().linear_forward(x, weight, bias, relu)
    if out is not None:
      return out
    _fallback("linear_forward")
  y = F.linear(x, weight, bias.to(x.dtype) if bias is not None else None)
  return torch.relu_(y) if relu else y


def linear_backward(backend, dy, x, weight, y, relu, need_dx, grad_w, grad_b, groups=1, group_stride=0):
  if backend == "native" and x.is_cuda:
    out = _native().linear_backward(dy, x, weight, y, relu, need_dx, grad_w, grad_b, groups, group_stride)
    if out is not NotImplemented:
      return out
    _fallback("linear_backward")
  if groups > 1:
    pieces = [linear_backward(backend, dy_g, x_g, weight, y_g, relu, need_dx, group_view(grad_w, g, group_stride), group_view(grad_b, g, group_stride))
              for g, (dy_g, x_g, y_g) in enumerate(zip(_chunks(dy, groups), _chunks(x, groups), _chunks(y, groups)))]
    return torch.cat(pieces, dim=0) if need_dx else None
  if relu:
    dy = _relu_mask(dy, y)
  grad_w.copy_(dy.t() @ x)
  if grad_b is not None:
    grad_b.copy_((dy if dy.dtype == torch.float64 else dy.float()).sum(dim=0))
  return dy @ weight if need_dx else None


# ---------------------------------------------------------------------------- #
# Batch normalisation

def batchnorm_forward(backend, x, gamma, beta, moving_mean, moving_var, decay, eps, relu, groups=1, coef=False):
  """Training-mode batch norm; with `groups` > 1 every consecutive batch slice (one logical worker) has its own statistics;
  returns (y, mean [groups * C], rstd [groups * C]), and with `coef` a fourth item: the native kernels' (scale, shift), what
  `batchnorm_backward(mask_coef=)` takes (None from the torch provider)."""
  if backend == "native" and x.is_cuda:
    out = _native().batchnorm_forward(x, gamma, beta, moving_mean, moving_var, decay, eps, relu, groups, coef=coef)
    if out is not None:
      return out
    _fallback("batchnorm_forward")
  if coef:
    return batchnorm_forward(backend, x, gamma, beta, moving_mean, moving_var, decay, eps, relu, groups) + (None,)
  if groups > 1:
    outs = [batchnorm_forward(backend, x_g.contiguous(memory_format=_CL), gamma, beta, moving_mean if g == 0 else None, moving_var if g == 0 else None, decay, eps, relu)
            for g, x_g in enumerate(_chunks(x, groups))]
    return torch.cat([o[0] for o in outs], dim=0).contiguous(memory_format=_CL), torch.cat([o[1] for o in outs]), torch.cat([o[2] for o in outs])
  y, mean, rstd = torch.native_batch_norm(x, gamma, beta, moving_mean, moving_var, True, 1.0 - decay, eps)
  if relu:
    y = torch.relu_(y)
  return y, mean, rstd


def batchnorm_add_relu_forward(backend, x, gamma, beta, moving_mean, moving_var, decay, eps, residual, groups=1):
  """y = relu(bn(x) + residual): the closing batch norm, shortcut add and ReLU of a residual unit in one pass. Returns (y, mean, rstd)."""
  if backend == "native" and x.is_cuda:
    out = _native().batchnorm_forward(x, gamma, beta, moving_mean, moving_var, decay, eps, True, groups, residual)
    if out is not None:
      return out
    _fallback("batchnorm_add_relu_forward")
  y, mean, rstd = batchnorm_forward(backend, x, gamma, beta, moving_mean, moving_var, decay, eps, False, groups)
  return add_relu_forward(backend, y, residual, True), mean, rstd


def batchnorm_add_relu_backward(backend, dy, x, y, gamma, mean, rstd, grad_gamma, grad_beta, groups=1, group_stride=0):
  """Backward of `batchnorm_add_relu_forward`: returns (dx, g) with g = dy * (y > 0), the gradient of the residual input."""
  if backend == "native" and x.is_cuda:
    out = _native().batchnorm_backward(dy, x, y, gamma, mean, rstd, True, grad_gamma, grad_beta, groups, group_stride, True)
    if out is not None:
      return out
    _fallback("batchnorm_add_relu_backward")
  g = relu_backward(backend, dy, y)
  return batchnorm_backward(backend, g, x, None, gamma, mean, rstd, False, grad_gamma, grad_beta, groups, group_stride), g


def batchnorm_inference(backend, x, gamma, beta, moving_mean, moving_var, eps, relu):
  y = F.batch_norm(x, moving_mean, moving_var, gamma, beta, False, 0.0, eps)
  return torch.relu_(y) if relu else y


def batchnorm_backward(backend, dy, x, y, gamma, mean, rstd, relu, grad_gamma, grad_beta, groups=1, group_stride=0, mask_coef=None):
  """`mask_coef`: the fourth item of `batchnorm_forward(coef=True)` for the forward that produced `y`, or None."""
  if backend == "native" and x.is_cuda:
    out = _native().batchnorm_backward(dy, x, y, gamma, mean, rstd, relu, grad_gamma, grad_beta, groups, group_stride, mask_coef=mask_coef)
    if out is not None:
      return out
    _fallback("batchnorm_backward")
  if groups > 1:
    c = x.shape[1]
    pieces = [batchnorm_backward(backend, dy_g.contiguous(memory_format=_CL), x_g.contiguous(memory_format=_CL), y_g, gamma, mean[g * c:(g + 1) * c], rstd[g * c:(g + 1) * c], relu,
                                 group_view(grad_gamma, g, group_stride), group_view(grad_beta, g, group_stride))
              for g, (dy_g, x_g, y_g) in enumerate(zip(_chunks(dy, groups), _chunks(x, groups), _chunks(y, groups)))]
    return torch.cat(pieces, dim=0).contiguous(memory_format=_CL)
  if relu:
    dy = _relu_mask(dy, y)
  # without gamma (slim `scale=False`) a unit weight is passed: the CUDA kernel returns an empty bias gradient for an undefined weight
  weight = gamma if gamma is not None else torch.ones(x.shape[1], dtype=mean.dtype, device=x.device)
  dx, dgamma, dbeta = torch.ops.aten.native_batch_norm_backward(dy, x, weight, None, None, mean, rstd, True, 1e-5, [True, gamma is not None, True])
  if grad_gamma is not None:
    grad_gamma.copy_(dgamma)
  grad_beta.copy_(dbeta)
  return dx


def layernorm_forward(backend, x, gamma, beta, eps):
  """LayerNorm over the last dimension of a [rows, C] tensor -> (y, mean[rows], rstd[rows])."""
  if backend == "native" and x.is_cuda:
    out = _native().layernorm_forward(x, gamma, beta, eps)
    if out is not None:
      return out
    _fallback("layernorm_forward")
  xf = x if x.dtype == torch.float64 else x.float()
  mean = xf.mean(dim=1)
  var = xf.var(dim=1, unbiased=False)
  rstd = torch.rsqrt(var + eps)
  y = (xf - mean[:, None]) * rstd[:, None] * gamma.to(xf.dtype) + beta.to(xf.dtype)
  return y.to(x.dtype), mean, rstd


def layernorm_backward(backend, dy, x, gamma, mean, rstd, grad_gamma, grad_beta, groups=1, group_stride=0):
  if groups > 1:
    rows = x.shape[0] // groups
    pieces = [layernorm_backward(backend, dy[g * rows:(g + 1) * rows], x[g * rows:(g + 1) * rows].contiguous(), gamma, mean[g * rows:(g + 1) * rows], rstd[g * rows:(g + 1) * rows],
                                 group_view(grad_gamma, g, group_stride), group_view(grad_beta, g, group_stride)) for g in range(groups)]
    return torch.cat(pieces, dim=0)
  if backend == "native" and x.is_cuda:
    out = _native().layernorm_backward(dy, x, gamma, mean, rstd, grad_gamma, grad_beta)
    if out is not None:
      return out
    _fallback("layernorm_backward")
  kind = x.dtype if x.dtype == torch.float64 else torch.float32
  xf, df = x.to(kind), dy.to(kind)
  xhat = (xf - mean.to(kind)[:, None]) * rstd.to(kind)[:, None]
  g = df * gamma.to(kind)
  grad_gamma.copy_((df * xhat).sum(dim=0))
  grad_beta.copy_(df.sum(dim=0))
  dx = rstd.to(kind)[:, None] * (g - g.mean(dim=1, keepdim=True) - xhat * (g * xhat).mean(dim=1, keepdim=True))
  return dx.to(x.dtype)


# ---------------------------------------------------------------------------- #
# Element-wise / pooling

def relu_forward(backend, x):
  return torch.relu(x)


def relu_backward(backend, dy, y):
  if backend == "native" and dy.is_cuda:
    out = _native().relu_backward(dy, y)
    if out is not None:
      return out
    _fallback("relu_backward")
  return _relu_mask(dy, y)


def add_relu_forward(backend, a, b, relu):
  if backend == "native" and a.is_cuda:
    out = _native().add_relu_forward(a, b, relu)
    if out is not None:
      return out
    _fallback("add_relu_forward")
  y = a + b
  return torch.relu_(y) if relu else y


def add_forward(backend, a, b):
  if a is None:
    return b
  if b is None:
    return a
  if backend == "native" and a.is_cuda:
    out = _native().add_relu_forward(a, b, False)
    if out is not None:
      return out
    _fallback("add_forward")
  return a + b


def maxpool_forward(backend, x, k, stride, pads):
  """Returns (y, index): `index` is the torch int64 argmax (library provider) or a uint8 window-relative argmax (native)."""
  if backend == "native" and x.is_cuda:
    out = _native().maxpool_forward(x, k, stride, pads)
    if out is not None:
      return out
    _fallback("maxpool_forward")
  t, b, l, r = pads
  xp = F.pad(x, (l, r, t, b), value=float("-inf")) if any(pads) else x
  y, index = F.max_pool2d(xp, k, stride, return_indices=True)
  return y, index


def maxpool_backward(backend, dy, shape, index, k, stride, pads, x, y):
  if index.dtype == torch.uint8:
    return _native().maxpool_backward(dy, shape, index, k, stride, pads)
  t, b, l, r = pads
  n, c, h, w = shape
  xp_shape = (n, c, h + t + b, w + l + r)
  dxp = torch.ops.aten.max_pool2d_with_indices_backward(dy, dy.new_empty(xp_shape).contiguous(memory_format=_CL), [k, k], [stride, stride], [0, 0], [1, 1], False, index)
  return dxp[:, :, t:t + h, l:l + w].contiguous(memory_format=_CL)


def avgpool2d_forward(backend, x, k, stride, pads):
  """Native k x k average pool with the TF "SAME" divisor, or None (the caller keeps its aten implementation)."""
  if backend == "native" and x.is_cuda:
    out = _native().avgpool2d_forward(x, k, stride, pads)
    if out is None:
      _fallback("avgpool2d_forward")
    return out
  return None


def avgpool2d_backward(backend, dy, shape, k, stride, pads):
  if backend == "native" and dy.is_cuda:
    out = _native().avgpool2d_backward(dy, shape, k, stride, pads)
    if out is None:
      _fallback("avgpool2d_backward")
    return out
  return None


def relu6_forward(backend, x):
  if backend == "native" and x.is_cuda:
    out = _native().relu6(x)
    if out is not None:
      return out
    _fallback("relu6_forward")
  return torch.clamp(x, 0.0, 6.0)


def relu6_backward(backend, dy, x):
  if backend == "native" and x.is_cuda:
    out = _native().relu6(x, dy)
    if out is not None:
      return out
    _fallback("relu6_backward")
  return dy * ((x > 0) & (x < 6)).to(dy.dtype)


def global_avgpool_forward(backend, x):
  if backend == "native" and x.is_cuda:
    out = _native().global_avgpool_forward(x)
    if out is not None:
      return out
    _fallback("global_avgpool_forward")
  return (x if x.dtype == torch.float64 else x.float()).mean(dim=(2, 3), keepdim=True).to(x.dtype)


def global_avgpool_backward(backend, dy, shape):
  n, c, h, w = shape
  if backend == "native" and dy.is_cuda:
    out = _native().global_avgpool_backward(dy, shape)
    if out is not None:
      return out
    _fallback("global_avgpool_backward")
  return (dy / (h * w)).expand(n, c, h, w).contiguous(memory_format=_CL)


def subsample_forward(backend, x, stride):
  if backend == "native" and x.is_cuda:
    out = _native().subsample_forward(x, stride)
    if out is not None:
      return out
    _fallback("subsample_forward")
  return x[:, :, ::stride, ::stride].contiguous(memory_format=_CL)


def subsample_accumulate(backend, dx, dy, stride):
  """dx + subsample_backward(dy), adding dy in place at the sampled pixels of dx (equal under `torch.equal`: a -0 of dx stays -0)."""
  if backend == "native" and dx.is_cuda:
    out = _native().subsample_accumulate(dx, dy, stride)
    if out is not None:
      return out
    _fallback("subsample_accumulate")
  return add_forward(backend, subsample_backward(backend, dy, dx.shape, stride), dx)


def subsample_backward(backend, dy, shape, stride):
  if backend == "native" and dy.is_cuda:
    out = _native().subsample_backward(dy, shape, stride)
    if out is not None:
      return out
    _fallback("subsample_backward")
  n, c, h, w = shape
  dx = torch.zeros((n, h, w, c), dtype=dy.dtype, device=dy.device).permute(0, 3, 1, 2)  # zeros allocated directly in NHWC memory
  dx[:, :, ::stride, ::stride] = dy
  return dx


# ---------------------------------------------------------------------------- #
# Loss

def flip_labels(labels, classes, groups=1, flip_from=0):
  """Labels of the label-flipping attack: y -> `classes` - 1 - y in the consecutive batch slices (groups) >= `flip_from`; a label outside
  [0, classes) matches no class and is left as it is."""
  if not 0 <= flip_from <= groups:
    raise ValueError("flip_from must lie in [0, groups] (got %r for %d groups)" % (flip_from, groups))
  lo = labels.shape[0] // groups * flip_from
  tail = labels[lo:]
  return torch.cat([labels[:lo], torch.where((tail >= 0) & (tail < classes), classes - 1 - tail, tail)])


def check_backdoor(backdoor, classes, groups, rows):
  """Validates a backdoor descriptor (first group, q, target, scale) for `groups` groups of `rows` rows and `classes` classes."""
  first, q, target, scale = backdoor
  if not (0 <= first <= groups and 0 <= q <= rows and 0 <= target < classes and math.isfinite(scale) and scale > 0.):
    raise ValueError("invalid backdoor descriptor %r for %d groups of %d rows and %d classes" % (tuple(backdoor), groups, rows, classes))


def backdoor_labels(labels, groups, first, q, target):
  """Labels of the backdoor attack: the first `q` rows of every consecutive batch slice (group) >= `first` become `target`."""
  rows = labels.shape[0] // groups
  out = labels.clone()
  for g in range(first, groups):
    out[g * rows:g * rows + q] = target
  return out


def softmax_xent(backend, logits, labels, label_smoothing=0.0, groups=1, flip_from=None, backdoor=None):
  """Mean softmax cross-entropy -> (loss, dlogits [B, K]). `groups` == 1: 0-d loss over the batch; `groups` > 1: one mean per
  consecutive batch slice (logical worker), loss of shape [groups], gradients scaled by 1 / (B / groups). `flip_from`: the groups
  >= flip_from train on `flip_labels` (label-flipping attack; None: no flip). A label outside [0, K) matches no class.
  `backdoor` = (first, q, target, scale): the groups >= first train on `backdoor_labels` and their dlogits are multiplied by `scale`;
  the loss is not (backdoor attack; None: no poisoning)."""
  if flip_from is not None and backdoor is not None:
    raise ValueError("label flipping and the backdoor are two attacks: give flip_from or backdoor, not both")
  if backdoor is not None:
    check_backdoor(backdoor, logits.shape[1], groups, logits.shape[0] // groups)
  if backend == "native" and logits.is_cuda:
    out = _native().softmax_xent(logits, labels, label_smoothing, groups, flip_from, backdoor)
    if out is not None:
      return out
    _fallback("softmax_xent")
  if flip_from is not None:
    labels = flip_labels(labels, logits.shape[1], groups, flip_from)
  if backdoor is not None:
    first, q, target, scale = backdoor
    loss, dlogits = softmax_xent(backend, logits, backdoor_labels(labels, groups, first, q, target), label_smoothing, groups)
    if scale != 1.0 and first < groups:
      rows = logits.shape[0] // groups
      dlogits = torch.cat([dlogits[:first * rows], dlogits[first * rows:] * scale])
    return loss, dlogits
  if groups > 1:
    outs = [softmax_xent(backend, lg, lb, label_smoothing) for lg, lb in zip(_chunks(logits, groups), _chunks(labels, groups))]
    return torch.stack([o[0] for o in outs]), torch.cat([o[1] for o in outs], dim=0)
  z = logits if logits.dtype == torch.float64 else logits.float()
  logp = torch.log_softmax(z, dim=1)
  batch, classes = z.shape
  target = (torch.arange(classes, device=z.device) == labels.view(-1, 1)).to(z.dtype)
  if label_smoothing > 0.:
    target = target * (1.0 - label_smoothing) + label_smoothing / classes
  loss = -(target * logp).sum(dim=1).mean()
  return loss, (torch.exp(logp) - target) / batch


# ---------------------------------------------------------------------------- #
# Input pipeline tail

_VGG_MEANS = (123.68, 116.78, 103.94)


def trigger_size(height, width):
  """Side s = ceil(min(H, W) / 10) of the backdoor trigger of an H x W network input (MNIST 3, CIFAR 4, 224-pixel ImageNet 23)."""
  s = -(-min(height, width) // 10)
  if s + 1 > min(height, width):
    raise ValueError("a %d x %d input has no room for the backdoor trigger" % (height, width))
  return s


def trigger_descriptor(images, trigger):
  """The kernels' descriptor (rows, first, q, s) of `trigger` = (groups, first, q) on the NHW[C] batch `images`."""
  groups, first, q = trigger
  n, h, w = images.shape[:3]
  if groups < 1 or n % groups or not (0 <= first and 0 <= q <= n // groups):
    raise ValueError("invalid backdoor trigger %r for a batch of %d images" % (tuple(trigger), n))
  return n // groups, first, q, trigger_size(h, w)


def stamp_trigger(images, groups, first, q):
  """The backdoor trigger on a raw NHW[C] batch in the [0, 255] domain (any dtype), as a new tensor: an s x s checkerboard
  (`trigger_size`), 255 where i + j is even and 0 elsewhere on every channel, at the bottom right one pixel from the edges (rows and
  columns H - 1 - s .. H - 2 and W - 1 - s .. W - 2), on the first `q` images of every consecutive slice of n / `groups` images from slice
  `first` on. The one definition of the pattern and its placement: the kernels (`Trigger` in `agb_device.cuh`) are tested against it."""
  rows, first, q, s = trigger_descriptor(images, (groups, first, q))
  h, w = images.shape[1:3]
  out = images.clone()
  for g in range(first, groups):
    patch = out[g * rows:g * rows + q, h - 1 - s:h - 1, w - 1 - s:w - 1]
    patch.fill_(0)
    patch[:, 0::2, 0::2] = 255
    patch[:, 1::2, 1::2] = 255
  return out


def image_normalize(backend, images, mode, dtype, trigger=None):
  """uint8 NHWC host-format batch (already on the device) -> normalised (N, C, H, W) channels_last activations.
  `vgg`: subtract the per-channel ImageNet means; `inception`: x/127.5 - 1; `lenet`: (x - 128)/128. `trigger` = (groups, first, q):
  the backdoor trigger on the images `stamp_trigger` poisons (None: none)."""
  if backend == "native" and images.is_cuda:
    out = _native().image_normalize(images, mode, dtype, trigger)
    if out is not None:
      return out
    _fallback("image_normalize")
  if trigger is not None:
    images = stamp_trigger(images, *trigger)
  x = images.to(torch.float32)
  if mode == "vgg" and x.shape[-1] == 3:
    x = x - torch.tensor(_VGG_MEANS, device=x.device)
  elif mode == "inception":
    x = x / 127.5 - 1.0
  else:
    x = (x - 128.0) / 128.0
  return x.to(dtype).permute(0, 3, 1, 2)  # NHWC memory viewed as (N, C, H, W): already channels_last

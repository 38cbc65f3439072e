"""Static layer graph with explicit forward/backward — the model-side execution engine.

The reference builds a TF1 static graph per worker replica and lets TF differentiate it
(`graph.py:254-273`). Here models are trees of `Module`s with hand-written `forward` and
`backward`, executed over pre-planned buffers:

* parameters are *views* into the flat fp32 master buffer (and its bf16 compute copy); a module
  never owns storage, so the aggregation kernel and the layers share memory with zero copies;
* `backward` writes each variable's gradient straight into the current worker's row of the
  peer-mapped gradient matrix (`ctx.grads[name]`), in fp32;
* no autograd tape, no tracing compiler: a step is a fixed sequence of kernel launches, which is
  what CUDA-graph capture wants.

Activations are NHWC in memory (torch shape (N, C, H, W) with channels_last strides), bf16 on
GPU / fp32 on CPU. Conv weights are OHWI in memory (K-major rows for the implicit-GEMM kernels).
Every op has two providers selected by `ctx.backend`: `"native"` = the hand-written sm_90a
kernels of `native/op_nn` (ops/nn.py), `"torch"` = aten library calls (cuDNN/cuBLAS) used as
the numerical reference and as the baseline arm.
"""

import math
import os

import torch
import torch.nn.functional as F

from ..ops import nn as nn_ops


class Context:
  """Per-execution state handed to every module."""

  def __init__(self, backend="torch", training=True, dtype=torch.float32, device="cpu"):
    self.backend = backend      # "native" | "torch"
    self.training = training
    self.dtype = dtype          # activation/compute dtype
    self.device = torch.device(device)
    self.weights = None         # name -> compute-dtype view of the parameters
    self.master = None          # name -> fp32 master view
    self.grads = None           # name -> fp32 gradient view of the current worker
    self.state = None           # name -> non-trainable state tensor (BN moving statistics)
    self.generator = None       # torch.Generator for dropout
    self.aux_heads = []         # `AuxHead`s that produced side logits during the current training forward
    self.need_input_grad = False
    self.backward_hook = None   # callable(layer) run by `Sequential.backward` after each child: gradient-bucket publication
    self.groups = 1             # logical workers batched in one pass (their batches are consecutive along dim 0)
    self.group_stride = 0       # elements between two workers' gradient rows (`grads` are worker 0's views)
    self.flip_from = None       # label-flipping attack: the groups >= flip_from train on the labels K - 1 - y (None: no flip)
    self.backdoor = None        # backdoor attack: (first group, q, target, scale): the first q images of every group >= first carry the
                                # trigger and train on `target`, the groups' loss gradients scaled by `scale` (None: no poisoning)


class Module:
  """Base layer: declares variables, runs forward, runs backward (storing what it needs in `self`)."""

  def __init__(self, name=None):
    self.name = name if name is not None else type(self).__name__.lower()

  def declare(self, layout, states):
    """Register trainable variables in `layout` (FlatLayout) and non-trainable ones in `states` (dict name -> shape)."""

  def initialize(self, master, states, generator):
    """Write initial values into the fp32 master views / state tensors."""

  def forward(self, x, ctx):
    raise NotImplementedError

  def backward(self, dy, ctx):
    raise NotImplementedError

  def children(self):
    return ()

  def release(self):
    """Drop tensors saved for backward."""
    for key in [k for k in self.__dict__ if k.startswith("_saved")]:
      self.__dict__[key] = None
    for child in self.children():
      child.release()


def _trunc_normal_(tensor, std, generator):
  torch.nn.init.trunc_normal_(tensor, mean=0.0, std=std, a=-2 * std, b=2 * std, generator=generator)


def _conv_out(size, k, stride, pad_lo, pad_hi):
  return (size + pad_lo + pad_hi - k) // stride + 1


def same_padding(size, k, stride):
  """TensorFlow 'SAME' padding -> (lo, hi)."""
  out = -(-size // stride)
  total = max((out - 1) * stride + k - size, 0)
  return total // 2, total - total // 2


class Conv2d(Module):
  """2-D convolution, NHWC / OHWI. `k`: int or (kh, kw) (the 1x7 / 7x1 / 1x3 / 3x1 factorised kernels of the Inception
  families). `padding`: "SAME" (TF semantics), "VALID", or anything else = symmetric explicit, the `conv2d_same` convention
  of slim's resnet_utils: pad (k-1)//2, k-1-(k-1)//2 then VALID."""

  def __init__(self, name, cin, cout, k, stride=1, padding="SAME", bias=False, relu=False, init="variance_scaling", init_std=None, bias_init=0.0):
    super().__init__(name)
    self.kh, self.kw = (k, k) if isinstance(k, int) else tuple(k)
    self.cin, self.cout, self.k, self.stride, self.padding = cin, cout, k, stride, padding
    self.bias, self.relu, self.init, self.init_std, self.bias_init = bias, relu, init, init_std, bias_init

  def declare(self, layout, states):
    layout.add(self.name + "/weights", (self.cout, self.kh, self.kw, self.cin))
    if self.bias:
      layout.add(self.name + "/biases", (self.cout,))

  def initialize(self, master, states, generator):
    w = master[self.name + "/weights"]
    fan_in = self.kh * self.kw * self.cin
    if self.init == "truncated_normal":
      _trunc_normal_(w, self.init_std, generator)
    elif self.init == "xavier":
      limit = math.sqrt(6.0 / (fan_in + self.kh * self.kw * self.cout))
      w.uniform_(-limit, limit, generator=generator)
    else:  # slim variance_scaling_initializer(): truncated normal, stddev = sqrt(2 / fan_in) / .8796...
      _trunc_normal_(w, math.sqrt(2.0 / fan_in) / 0.87962566103423978, generator)
    if self.bias:
      master[self.name + "/biases"].fill_(self.bias_init)

  def _pads(self, h, w):
    if self.padding == "SAME":
      return same_padding(h, self.kh, self.stride) + same_padding(w, self.kw, self.stride)
    if self.padding == "VALID":
      return (0, 0, 0, 0)
    th, tw = self.kh - 1, self.kw - 1
    return (th // 2, th - th // 2, tw // 2, tw - tw // 2)

  def forward(self, x, ctx):
    n, c, h, w = x.shape
    pads = self._pads(h, w)
    weight = ctx.weights[self.name + "/weights"]
    bias = ctx.master[self.name + "/biases"] if self.bias else None
    aux = {} if ctx.training else None
    y = nn_ops.conv2d_forward(ctx.backend, x, weight, bias, self.stride, pads, self.relu, aux)
    if ctx.training:
      self._saved_x, self._saved_y, self._saved_pads, self._saved_aux = x, (y if self.relu else None), pads, aux
    return y

  def backward(self, dy, ctx, addend=None):
    """`addend` (the input's shape): returns dx + addend (a gradient reaching the same input by another path)."""
    x, pads = self._saved_x, self._saved_pads
    weight = ctx.weights[self.name + "/weights"]
    need_dx = ctx.need_input_grad or not getattr(self, "is_first", False) or addend is not None
    dx, dw, db = nn_ops.conv2d_backward(ctx.backend, dy, x, weight, self._saved_y, self.stride, pads, self.relu, self.bias, need_dx,
                                        ctx.grads[self.name + "/weights"], ctx.grads[self.name + "/biases"] if self.bias else None, ctx.groups, ctx.group_stride,
                                        self._saved_aux, addend)
    self._saved_x = self._saved_y = self._saved_aux = None
    return dx


class Dense(Module):
  """Fully connected layer y = x W^T + b, W stored [out, in] (K-major rows)."""

  def __init__(self, name, fin, fout, relu=False, bias=True, init="xavier", init_std=None, bias_init=0.0):
    super().__init__(name)
    self.fin, self.fout, self.relu, self.bias, self.init, self.init_std, self.bias_init = fin, fout, relu, bias, init, init_std, bias_init

  def declare(self, layout, states):
    layout.add(self.name + "/weights", (self.fout, self.fin))
    if self.bias:
      layout.add(self.name + "/biases", (self.fout,))

  def initialize(self, master, states, generator):
    w = master[self.name + "/weights"]
    if self.init == "truncated_normal":
      _trunc_normal_(w, self.init_std, generator)
    else:  # glorot uniform: tf.get_variable's default initializer (reference: experiments/mnist.py:95-96)
      limit = math.sqrt(6.0 / (self.fin + self.fout))
      w.uniform_(-limit, limit, generator=generator)
    if self.bias:
      master[self.name + "/biases"].fill_(self.bias_init)

  def forward(self, x, ctx):
    x = x.reshape(x.shape[0], -1)
    weight = ctx.weights[self.name + "/weights"]
    bias = ctx.master[self.name + "/biases"] if self.bias else None
    y = nn_ops.linear_forward(ctx.backend, x, weight, bias, self.relu)
    if ctx.training:
      self._saved_x, self._saved_y = x, (y if self.relu else None)
    return y

  def backward(self, dy, ctx):
    need_dx = ctx.need_input_grad or not getattr(self, "is_first", False)
    dx = nn_ops.linear_backward(ctx.backend, dy, self._saved_x, ctx.weights[self.name + "/weights"], self._saved_y, self.relu, need_dx,
                                ctx.grads[self.name + "/weights"], ctx.grads[self.name + "/biases"] if self.bias else None, ctx.groups, ctx.group_stride)
    self._saved_x = self._saved_y = None
    return dx


class BatchNorm(Module):
  """Batch normalisation over (N, H, W) per channel with trainable gamma/beta and moving statistics
  (slim `batch_norm`: decay 0.997, epsilon 1e-5, scale=True in `resnet_arg_scope`), optionally fused with ReLU."""

  def __init__(self, name, channels, relu=False, decay=0.997, epsilon=1e-5, scale=True):
    super().__init__(name)
    self.channels, self.relu, self.decay, self.epsilon, self.scale = channels, relu, decay, epsilon, scale

  def declare(self, layout, states):
    if self.scale:
      layout.add(self.name + "/gamma", (self.channels,))
    layout.add(self.name + "/beta", (self.channels,))
    states[self.name + "/moving_mean"] = (self.channels,)
    states[self.name + "/moving_variance"] = (self.channels,)

  def initialize(self, master, states, generator):
    if self.scale:
      master[self.name + "/gamma"].fill_(1.0)
    master[self.name + "/beta"].zero_()
    states[self.name + "/moving_mean"].zero_()
    states[self.name + "/moving_variance"].fill_(1.0)

  def forward(self, x, ctx):
    gamma = ctx.master[self.name + "/gamma"] if self.scale else None
    beta = ctx.master[self.name + "/beta"]
    mean, var = ctx.state[self.name + "/moving_mean"], ctx.state[self.name + "/moving_variance"]
    if not ctx.training:
      return nn_ops.batchnorm_inference(ctx.backend, x, gamma, beta, mean, var, self.epsilon, self.relu)
    # with ReLU, the coefficients applied let the backward recompute the mask y > 0 from x instead of reading y
    y, batch_mean, batch_rstd, coef = nn_ops.batchnorm_forward(ctx.backend, x, gamma, beta, mean, var, self.decay, self.epsilon, self.relu, ctx.groups, coef=True)
    self._saved = (x, y if self.relu else None, batch_mean, batch_rstd, coef if self.relu else None)
    return y

  def backward(self, dy, ctx):
    x, y, batch_mean, batch_rstd, coef = self._saved
    gamma = ctx.master[self.name + "/gamma"] if self.scale else None
    dx = nn_ops.batchnorm_backward(ctx.backend, dy, x, y, gamma, batch_mean, batch_rstd, self.relu,
                                   ctx.grads[self.name + "/gamma"] if self.scale else None, ctx.grads[self.name + "/beta"], ctx.groups, ctx.group_stride, mask_coef=coef)
    self._saved = None
    return dx

  # -- closing layer of a residual unit: y = relu(bn(x) + shortcut) in one pass ------------------------------------------ #
  def forward_add_relu(self, x, shortcut, ctx):
    gamma = ctx.master[self.name + "/gamma"] if self.scale else None
    beta = ctx.master[self.name + "/beta"]
    mean, var = ctx.state[self.name + "/moving_mean"], ctx.state[self.name + "/moving_variance"]
    if not ctx.training:
      return nn_ops.add_relu_forward(ctx.backend, nn_ops.batchnorm_inference(ctx.backend, x, gamma, beta, mean, var, self.epsilon, False), shortcut, True)
    y, batch_mean, batch_rstd = nn_ops.batchnorm_add_relu_forward(ctx.backend, x, gamma, beta, mean, var, self.decay, self.epsilon, shortcut, ctx.groups)
    self._saved = (x, y, batch_mean, batch_rstd)
    return y

  def backward_add_relu(self, dy, ctx):
    """-> (gradient of x, gradient of the shortcut input)."""
    x, y, batch_mean, batch_rstd = self._saved
    gamma = ctx.master[self.name + "/gamma"] if self.scale else None
    self._saved = None
    return nn_ops.batchnorm_add_relu_backward(ctx.backend, dy, x, y, gamma, batch_mean, batch_rstd, ctx.grads[self.name + "/gamma"] if self.scale else None,
                                              ctx.grads[self.name + "/beta"], ctx.groups, ctx.group_stride)


class LayerNorm(Module):
  """Layer normalisation over the feature dimension of a [rows, features] activation (trainable gamma / beta)."""

  def __init__(self, name, features, epsilon=1e-5):
    super().__init__(name)
    self.features, self.epsilon = features, epsilon

  def declare(self, layout, states):
    layout.add(self.name + "/gamma", (self.features,))
    layout.add(self.name + "/beta", (self.features,))

  def initialize(self, master, states, generator):
    master[self.name + "/gamma"].fill_(1.0)
    master[self.name + "/beta"].zero_()

  def forward(self, x, ctx):
    x = x.reshape(x.shape[0], -1)
    y, mean, rstd = nn_ops.layernorm_forward(ctx.backend, x, ctx.master[self.name + "/gamma"], ctx.master[self.name + "/beta"], self.epsilon)
    if ctx.training:
      self._saved = (x, mean, rstd)
    return y

  def backward(self, dy, ctx):
    x, mean, rstd = self._saved
    self._saved = None
    return nn_ops.layernorm_backward(ctx.backend, dy, x, ctx.master[self.name + "/gamma"], mean, rstd, ctx.grads[self.name + "/gamma"], ctx.grads[self.name + "/beta"],
                                     ctx.groups, ctx.group_stride)


class ReLU(Module):
  def forward(self, x, ctx):
    y = nn_ops.relu_forward(ctx.backend, x)
    if ctx.training:
      self._saved_y = y
    return y

  def backward(self, dy, ctx):
    dx = nn_ops.relu_backward(ctx.backend, dy, self._saved_y)
    self._saved_y = None
    return dx


class MaxPool(Module):
  """Max pooling; `padding` "SAME" / "VALID" (TF semantics; SAME pads with -inf)."""

  def __init__(self, name, k, stride, padding="VALID"):
    super().__init__(name)
    self.k, self.stride, self.padding = k, stride, padding

  def forward(self, x, ctx):
    n, c, h, w = x.shape
    pads = (same_padding(h, self.k, self.stride) + same_padding(w, self.k, self.stride)) if self.padding == "SAME" else (0, 0, 0, 0)
    y, index = nn_ops.maxpool_forward(ctx.backend, x, self.k, self.stride, pads)
    if ctx.training:
      self._saved = (x.shape, index, pads, x, y)
    return y

  def backward(self, dy, ctx):
    shape, index, pads, x, y = self._saved
    self._saved = None
    return nn_ops.maxpool_backward(ctx.backend, dy, shape, index, self.k, self.stride, pads, x, y)


class GlobalAvgPool(Module):
  """Mean over H, W keeping a 1x1 map (slim `pool5`)."""

  def forward(self, x, ctx):
    self._saved_shape = x.shape
    return nn_ops.global_avgpool_forward(ctx.backend, x)

  def backward(self, dy, ctx):
    return nn_ops.global_avgpool_backward(ctx.backend, dy, self._saved_shape)


class AvgPool(Module):
  """Average pooling, "VALID" or TF "SAME" (padded positions are excluded from the divisor, as `tf.nn.avg_pool` does)."""

  def __init__(self, name, k, stride, padding="VALID"):
    super().__init__(name)
    self.k, self.stride, self.padding = k, stride, padding
    self._counts = {}

  def _count(self, h, w, pads, like):
    key = (h, w, like.dtype, like.device)
    if key not in self._counts:
      ones = F.pad(torch.ones((1, 1, h, w), dtype=torch.float32, device=like.device), (pads[2], pads[3], pads[0], pads[1]))
      self._counts[key] = (1.0 / F.avg_pool2d(ones, self.k, self.stride, divisor_override=1)).to(like.dtype)
    return self._counts[key]

  def forward(self, x, ctx):
    n, c, h, w = x.shape
    pads = (same_padding(h, self.k, self.stride) + same_padding(w, self.k, self.stride)) if self.padding == "SAME" else (0, 0, 0, 0)
    native = nn_ops.avgpool2d_forward(ctx.backend, x, self.k, self.stride, pads)
    if native is not None:
      self._saved = (tuple(x.shape), None, pads)
      return native
    xp = F.pad(x, (pads[2], pads[3], pads[0], pads[1])) if any(pads) else x
    self._saved = (xp.shape, (h, w), pads)
    y = F.avg_pool2d(xp, self.k, self.stride, divisor_override=1) * self._count(h, w, pads, x)
    return y.contiguous(memory_format=torch.channels_last)

  def backward(self, dy, ctx):
    shape, size, pads = self._saved
    if size is None:
      return nn_ops.avgpool2d_backward(ctx.backend, dy, shape, self.k, self.stride, pads)
    h, w = size
    dy = (dy * self._count(h, w, pads, dy)).contiguous(memory_format=torch.channels_last)
    proto = torch.empty(shape, dtype=dy.dtype, device=dy.device, memory_format=torch.channels_last)
    dxp = torch.ops.aten.avg_pool2d_backward(dy, proto, [self.k, self.k], [self.stride, self.stride], [0, 0], False, True, 1)
    return dxp[:, :, pads[0]:pads[0] + h, pads[2]:pads[2] + w].contiguous(memory_format=torch.channels_last)


class Subsample(Module):
  """slim `resnet_utils.subsample`: 1x1 max-pool with stride s == strided slicing."""

  def __init__(self, name, stride):
    super().__init__(name)
    self.stride = stride

  def forward(self, x, ctx):
    if self.stride == 1:
      return x
    self._saved_shape = x.shape
    return nn_ops.subsample_forward(ctx.backend, x, self.stride)

  def backward(self, dy, ctx):
    if self.stride == 1:
      return dy
    return nn_ops.subsample_backward(ctx.backend, dy, self._saved_shape, self.stride)


class Dropout(Module):
  def __init__(self, name, keep_prob):
    super().__init__(name)
    self.keep_prob = keep_prob

  def forward(self, x, ctx):
    if not ctx.training or self.keep_prob >= 1.0:
      self._saved_mask = None
      return x
    mask = (torch.rand(x.shape, device=x.device, generator=ctx.generator) < self.keep_prob).to(x.dtype) / self.keep_prob
    self._saved_mask = mask
    return x * mask

  def backward(self, dy, ctx):
    mask, self._saved_mask = self._saved_mask, None
    return dy if mask is None else dy * mask


class Flatten(Module):
  """NHWC flatten: (N, C, H, W) channels_last -> (N, H*W*C), matching TF's reshape of an NHWC tensor."""

  def forward(self, x, ctx):
    self._saved_shape = x.shape
    if x.dim() == 4:
      return x.permute(0, 2, 3, 1).reshape(x.shape[0], -1)
    return x.reshape(x.shape[0], -1)

  def backward(self, dy, ctx):
    shape = self._saved_shape
    if len(shape) == 4:
      n, c, h, w = shape
      return dy.reshape(n, h, w, c).permute(0, 3, 1, 2)
    return dy.reshape(shape)


class Sequential(Module):
  def __init__(self, name, layers):
    super().__init__(name)
    self.layers = list(layers)

  def children(self):
    return self.layers

  def declare(self, layout, states):
    for layer in self.layers:
      layer.declare(layout, states)

  def initialize(self, master, states, generator):
    for layer in self.layers:
      layer.initialize(master, states, generator)

  def forward(self, x, ctx):
    for layer in self.layers:
      x = layer.forward(x, ctx)
    return x

  def backward(self, dy, ctx):
    hook = ctx.backward_hook
    for layer in reversed(self.layers):
      dy = layer.backward(dy, ctx)
      if hook is not None:
        hook(layer)   # every gradient of `layer` (and of everything after it) has been written: see `Manager._plan_buckets`
    return dy


class Residual(Module):
  """y = relu(shortcut(x) + residual(x)) (ResNet v1 unit) or shortcut(x) + residual(x) (`relu=False`)."""

  def __init__(self, name, shortcut, residual, relu=True):
    super().__init__(name)
    self.shortcut, self.residual, self.relu = shortcut, residual, relu

  def children(self):
    return (self.shortcut, self.residual)

  def declare(self, layout, states):
    self.shortcut.declare(layout, states)
    self.residual.declare(layout, states)

  def initialize(self, master, states, generator):
    self.shortcut.initialize(master, states, generator)
    self.residual.initialize(master, states, generator)

  def _closing_norm(self):
    """The residual branch's last layer when the unit ends with BN -> add -> ReLU (ResNet v1): those three fuse into one pass."""
    if not self.relu or not isinstance(self.residual, Sequential) or not self.residual.layers or os.environ.get("AGB_FUSE_RESIDUAL", "1") == "0":
      return None
    last = self.residual.layers[-1]
    return last if (isinstance(last, BatchNorm) and not last.relu) else None

  def forward(self, x, ctx):
    a = self.shortcut.forward(x, ctx)
    norm = self._closing_norm()
    if norm is not None:
      b = x
      for layer in self.residual.layers[:-1]:
        b = layer.forward(b, ctx)
      return norm.forward_add_relu(b, a, ctx)
    b = self.residual.forward(x, ctx)
    y = nn_ops.add_relu_forward(ctx.backend, a, b, self.relu)
    if ctx.training and self.relu:
      self._saved_y = y
    return y

  def backward(self, dy, ctx):
    norm = self._closing_norm()
    if norm is not None:
      db, dy = norm.backward_add_relu(dy, ctx)
      if ctx.backend == "native" and isinstance(self.residual.layers[0], Conv2d) and len(self.residual.layers) > 2:
        return self._backward_summed(db, dy, ctx)
      for layer in reversed(self.residual.layers[:-1]):
        db = layer.backward(db, ctx)
      da = self.shortcut.backward(dy, ctx)
      return nn_ops.add_forward(ctx.backend, da, db)
    if self.relu:
      dy = nn_ops.relu_backward(ctx.backend, dy, self._saved_y)
      self._saved_y = None
    da = self.shortcut.backward(dy, ctx)
    db = self.residual.backward(dy, ctx)
    return nn_ops.add_forward(ctx.backend, da, db)


  def _backward_summed(self, db, dy, ctx):
    """Backward below the closing norm with the two gradients of x summed where the residual branch's first convolution writes its
    data gradient (the epilogue of a 1x1 stride-1 one), instead of by a separate pass over a tensor the size of x. A strided
    `Subsample` shortcut is added in place at the sampled pixels only. Same values as `add_forward(da, db)` under `torch.equal`."""
    strided = isinstance(self.shortcut, Subsample) and self.shortcut.stride > 1
    da = None if strided else self.shortcut.backward(dy, ctx)
    for layer in reversed(self.residual.layers[1:-1]):
      db = layer.backward(db, ctx)
    dx = self.residual.layers[0].backward(db, ctx, addend=da)
    return nn_ops.subsample_accumulate(ctx.backend, dx, dy, self.shortcut.stride) if strided else dx


class Identity(Module):
  def forward(self, x, ctx):
    return x

  def backward(self, dy, ctx):
    return dy


class Branches(Module):
  """Run several branches on the same input and concatenate along channels (Inception-style blocks)."""

  def __init__(self, name, branches):
    super().__init__(name)
    self.branches = list(branches)

  def children(self):
    return self.branches

  def declare(self, layout, states):
    for branch in self.branches:
      branch.declare(layout, states)

  def initialize(self, master, states, generator):
    for branch in self.branches:
      branch.initialize(master, states, generator)

  def forward(self, x, ctx):
    outs = [branch.forward(x, ctx) for branch in self.branches]
    self._saved_split = [o.shape[1] for o in outs]
    return torch.cat(outs, dim=1).contiguous(memory_format=torch.channels_last)

  def backward(self, dy, ctx):
    total = None
    for branch, piece in zip(self.branches, torch.split(dy, self._saved_split, dim=1)):
      dx = branch.backward(piece.contiguous(memory_format=torch.channels_last), ctx)
      total = dx if total is None else total + dx
    return total


class DepthwiseConv2d(Module):
  """Depthwise k x k convolution (TF "SAME" padding), `multiplier` output channels per input channel (slim
  `separable_conv2d(..., depth_multiplier)` first half). Weights [C * multiplier, k, k, 1]. A depthwise filter has no GEMM shape to
  put on the tensor cores: bandwidth kernels in `native/op_nn/depthwise.cu`, aten otherwise."""

  def __init__(self, name, channels, k, stride, multiplier=1, init_std=0.09):
    super().__init__(name)
    self.channels, self.k, self.stride, self.multiplier, self.init_std = channels, k, stride, multiplier, init_std

  def declare(self, layout, states):
    layout.add(self.name + "/depthwise_weights", (self.channels * self.multiplier, self.k, self.k, 1))

  def initialize(self, master, states, generator):
    _trunc_normal_(master[self.name + "/depthwise_weights"], self.init_std, generator)

  def forward(self, x, ctx):
    n, c, h, w = x.shape
    pads = same_padding(h, self.k, self.stride) + same_padding(w, self.k, self.stride)
    if ctx.training:
      self._saved = (x, pads)
    return nn_ops.depthwise_forward(ctx.backend, x, ctx.weights[self.name + "/depthwise_weights"], self.stride, pads)

  def backward(self, dy, ctx):
    x, pads = self._saved
    self._saved = None
    return nn_ops.depthwise_backward(ctx.backend, dy, x, ctx.weights[self.name + "/depthwise_weights"], self.stride, pads, ctx.grads[self.name + "/depthwise_weights"],
                                     ctx.groups, ctx.group_stride)


class ReLU6(Module):
  def forward(self, x, ctx):
    self._saved_x = x
    return nn_ops.relu6_forward(ctx.backend, x)

  def backward(self, dy, ctx):
    x, self._saved_x = self._saved_x, None
    return nn_ops.relu6_backward(ctx.backend, dy, x)


class Scale(Module):
  """y = factor * x (residual scaling of Inception-ResNet blocks)."""

  def __init__(self, name, factor):
    super().__init__(name)
    self.factor = factor

  def forward(self, x, ctx):
    return x * self.factor

  def backward(self, dy, ctx):
    return dy * self.factor


class OffsetSubsample(Module):
  """y[i, j] = x[stride * i + offset, stride * j + offset] (zero beyond the border), output ceil(size / stride): the
  zero-pad + crop + 1x1 strided average pool of NASNet's `factorized_reduction` second path."""

  def __init__(self, name, stride=2, offset=1):
    super().__init__(name)
    self.stride, self.offset = stride, offset

  def forward(self, x, ctx):
    n, c, h, w = x.shape
    self._saved_shape = x.shape
    oh, ow = -(-h // self.stride), -(-w // self.stride)
    picked = x[:, :, self.offset::self.stride, self.offset::self.stride]
    if picked.shape[2] == oh and picked.shape[3] == ow:
      return picked.contiguous(memory_format=torch.channels_last)
    y = torch.zeros((n, c, oh, ow), dtype=x.dtype, device=x.device).contiguous(memory_format=torch.channels_last)
    y[:, :, :picked.shape[2], :picked.shape[3]] = picked
    return y

  def backward(self, dy, ctx):
    n, c, h, w = self._saved_shape
    dx = torch.zeros((n, c, h, w), dtype=dy.dtype, device=dy.device).contiguous(memory_format=torch.channels_last)
    target = dx[:, :, self.offset::self.stride, self.offset::self.stride]
    target.copy_(dy[:, :, :target.shape[2], :target.shape[3]])
    return dx


class DropPath(Module):
  """Training-time stochastic depth on a cell branch (NASNet `_apply_drop_path`): each sample of the batch keeps the branch with
  probability `keep_prob` (scaled by 1 / keep_prob). The cell-depth scaling of the drop rate is folded into `keep_prob` by
  the model builder; the reference's additional training-progress scaling needs the total step count and is not applied."""

  def __init__(self, name, keep_prob):
    super().__init__(name)
    self.keep_prob = keep_prob

  def forward(self, x, ctx):
    if not ctx.training or self.keep_prob >= 1.0:
      self._saved_mask = None
      return x
    mask = (torch.rand((x.shape[0], 1, 1, 1), device=x.device, generator=ctx.generator) < self.keep_prob).to(x.dtype) / self.keep_prob
    self._saved_mask = mask
    return x * mask

  def backward(self, dy, ctx):
    mask, self._saved_mask = self._saved_mask, None
    return dy if mask is None else dy * mask


class Add(Module):
  """Multi-input node of a `Graph`: element-wise sum of its inputs."""

  multi_input = True

  def forward(self, xs, ctx):
    self._saved_count = len(xs)
    total = xs[0]
    for x in xs[1:]:
      total = nn_ops.add_forward(ctx.backend, total, x)
    return total

  def backward(self, dy, ctx):
    return [dy] * self._saved_count


class Concat(Module):
  """Multi-input node of a `Graph`: channel concatenation."""

  multi_input = True

  def forward(self, xs, ctx):
    self._saved_split = [x.shape[1] for x in xs]
    return torch.cat(xs, dim=1).contiguous(memory_format=torch.channels_last)

  def backward(self, dy, ctx):
    return [piece.contiguous(memory_format=torch.channels_last) for piece in torch.split(dy, self._saved_split, dim=1)]


class Graph(Module):
  """Static DAG of modules (NASNet / PNASNet cells, where a hidden state feeds several later nodes).

  Values are numbered: 0 .. `nb_inputs`-1 are the graph inputs, node i (in list order = a topological order) produces value
  `nb_inputs + i`. `nodes` = [(module, input_ids)]; a module flagged `multi_input` receives the list of its inputs and returns
  a list of input gradients, any other module takes exactly one input. The output is value `output` (default: the last one).
  Backward walks the nodes in reverse and sums the gradients of a value consumed several times.
  With `nb_inputs` == 1, forward takes the tensor itself; otherwise a list."""

  def __init__(self, name, nodes, nb_inputs=1, output=None):
    super().__init__(name)
    self.nodes = [(module, tuple(inputs)) for module, inputs in nodes]
    self.nb_inputs = nb_inputs
    self.output = output if output is not None else nb_inputs + len(self.nodes) - 1
    self.multi_input = nb_inputs > 1

  def children(self):
    return [module for module, _ in self.nodes]

  def declare(self, layout, states):
    for module, _ in self.nodes:
      module.declare(layout, states)

  def initialize(self, master, states, generator):
    for module, _ in self.nodes:
      module.initialize(master, states, generator)

  def forward(self, x, ctx):
    values = list(x) if self.nb_inputs > 1 else [x]
    for module, inputs in self.nodes:
      if getattr(module, "multi_input", False):
        values.append(module.forward([values[i] for i in inputs], ctx))
      else:
        values.append(module.forward(values[inputs[0]], ctx))
    return values[self.output]

  def backward(self, dy, ctx):
    grads = {self.output: dy}
    for index in range(len(self.nodes) - 1, -1, -1):
      module, inputs = self.nodes[index]
      g = grads.pop(self.nb_inputs + index, None)
      if g is None:  # value never used downstream of the output
        continue
      back = module.backward(g, ctx)
      if not getattr(module, "multi_input", False):
        back = [back]
      for i, gi in zip(inputs, back):
        if gi is None:
          continue
        grads[i] = gi if i not in grads else nn_ops.add_forward(ctx.backend, grads[i], gi)
    if self.nb_inputs > 1:
      return [grads.get(i) for i in range(self.nb_inputs)]
    return grads.get(0)


class AuxHead(Module):
  """Auxiliary classifier tapped off the trunk (Inception v3/v4, Inception-ResNet-v2, NASNet, PNASNet): the trunk activation
  passes through unchanged; in training the side `head` produces extra logits whose softmax cross-entropy enters the loss with
  `weight` (reference: `experiments/slims.py:122-125`, 0.4 x aux loss). The model's loss head fills `_saved_dlogits`."""

  def __init__(self, name, head, weight=0.4):
    super().__init__(name)
    self.head, self.weight = head, weight

  def children(self):
    return (self.head,)

  def declare(self, layout, states):
    self.head.declare(layout, states)

  def initialize(self, master, states, generator):
    self.head.initialize(master, states, generator)

  def forward(self, x, ctx):
    if ctx.training:
      logits = self.head.forward(x, ctx)
      self._saved_shape = logits.shape
      self._saved_logits = logits.reshape(logits.shape[0], -1)
      ctx.aux_heads.append(self)
    return x

  def backward(self, dy, ctx):
    dlogits, self._saved_dlogits, self._saved_logits = self._saved_dlogits, None, None
    dx = self.head.backward(dlogits, ctx)
    return nn_ops.add_forward(ctx.backend, dy, dx)


class Model:
  """A root module + input description + loss head."""

  def __init__(self, name, root, input_shape, num_classes, label_smoothing=0.0, aux=None):
    self.name, self.root, self.input_shape, self.num_classes = name, root, tuple(input_shape), num_classes
    self.label_smoothing = label_smoothing
    first = self._first_layer(root)
    if first is not None:
      first.is_first = True

  @staticmethod
  def _first_layer(module):
    while True:
      kids = list(module.children())
      if not kids:
        return module if isinstance(module, (Conv2d, Dense)) else None
      if isinstance(module, (Residual, Branches, Graph)):
        return None
      module = kids[0]

  def declare(self, layout, states):
    self.root.declare(layout, states)

  def initialize(self, master, states, generator):
    self.root.initialize(master, states, generator)

  def logits(self, x, ctx):
    ctx.aux_heads = []
    y = self.root.forward(x, ctx)
    self._raw_shape = y.shape
    return y.reshape(y.shape[0], -1)

  def loss_and_backward(self, x, labels, ctx):
    """Forward, mean softmax cross-entropy, backward. Returns the loss (0-d fp32 tensor; shape [ctx.groups] when several logical
    workers are batched: each worker's loss is the mean over its own slice of the batch). The groups >= `ctx.flip_from` train on
    flipped labels, and the groups `ctx.backdoor` poisons on the backdoor's target, in the main and the auxiliary heads alike."""
    logits = self.logits(x, ctx)
    loss, dlogits = nn_ops.softmax_xent(ctx.backend, logits, labels, self.label_smoothing, ctx.groups, ctx.flip_from, ctx.backdoor)
    dlogits = self._shaped(dlogits, self._raw_shape, ctx)
    for aux in ctx.aux_heads:
      aux_loss, aux_dlogits = nn_ops.softmax_xent(ctx.backend, aux._saved_logits, labels, self.label_smoothing, ctx.groups, ctx.flip_from, ctx.backdoor)
      loss = loss + aux.weight * aux_loss
      aux._saved_dlogits = self._shaped(aux_dlogits * aux.weight, aux._saved_shape, ctx)
    ctx.aux_heads = []
    self.root.backward(dlogits, ctx)
    return loss

  @staticmethod
  def _shaped(dlogits, shape, ctx):
    dlogits = dlogits.to(ctx.dtype).reshape(shape)
    return dlogits.contiguous(memory_format=torch.channels_last) if dlogits.dim() == 4 else dlogits

  def accuracy(self, x, labels, ctx):
    logits = self.logits(x, ctx)
    return (logits.float().argmax(dim=1) == labels).float().mean()

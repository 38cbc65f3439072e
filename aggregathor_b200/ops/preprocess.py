"""slim preprocessing on the device (reference: `external/slim/preprocessing/preprocessing_factory.py:64` -> slim's
`vgg_preprocessing`, `inception_preprocessing`, `cifarnet_preprocessing`, `lenet_preprocessing`, as used by
`experiments/slims.py:100-111` and `experiments/cnnet.py:123-130`).

`Preprocessor(mode, out_size, channels)` turns a uint8 NHWC batch at its storage resolution into network-resolution
activations: one launch of `native/op_nn/preprocess.cu` on CUDA, the same arithmetic in vectorised torch ops elsewhere.
Both draw their per-image random parameters from the same counter-based hash (seed, step counter, image index, slot), so
a CPU run and a GPU run of the same experiment see the same crops / flips / colour factors, and the step counter lives in a
device tensor: augmentation is replayable from a CUDA graph.

Modes (training / evaluation):
  vgg        short side -> r ~ U{256..512}, random crop, mirror, mean subtraction   /  r = 256, central crop
  inception  distorted bbox crop (area 5-100 %, aspect 3/4-4/3), resize, mirror, colour distortion, [-1, 1]  /  central 87.5 % + resize
  cifarnet   pad 4, random crop, mirror, brightness 63, contrast [0.2, 1.8], per-image standardisation  /  central crop + standardisation
  plain      (x - mean) * scale after a resize of the whole image (`lenet`: (x - 128) / 128)

`trigger` = (groups, first, q) writes the backdoor trigger (`ops.nn.stamp_trigger`) on the poisoned images, in the sampled pixels: after
the geometric operations and before every photometric one.
"""

import ctypes
import math

import numpy as np
import torch

MODES = {"plain": 0, "vgg": 1, "inception": 2, "cifarnet": 3}
_VGG_MEANS = (123.68, 116.78, 103.94)
_M64 = (1 << 64) - 1


def uniform01(seed, step, images, slot):
  """The kernel's counter-based uniform [0, 1): numpy uint64 replica of `uniform01` in `preprocess.cu`."""
  with np.errstate(over="ignore"):
    images = np.asarray(images, dtype=np.uint64)
    h = np.uint64(seed & _M64) ^ np.uint64((step * 0x9E3779B97F4A7C15) & _M64) ^ (((images << np.uint64(32)) | np.uint64(slot)) * np.uint64(0xD1B54A32D192ED03))
    h ^= h >> np.uint64(33)
    h *= np.uint64(0xff51afd7ed558ccd)
    h ^= h >> np.uint64(33)
    h *= np.uint64(0xc4ceb9fe1a85ec53)
    h ^= h >> np.uint64(33)
  return (h >> np.uint64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)


class Preprocessor:
  """Callable `(images uint8 [N, SH, SW, C] on any device, dtype, training) -> (N, C, OH, OW) channels_last activations`."""

  def __init__(self, mode, out_size, resize_min=256, resize_max=512, area=(0.05, 1.0), pad=4, mean=None, scale=1.0, seed=0):
    if mode not in MODES:
      raise ValueError("unknown preprocessing " + repr(mode))
    self.mode, self.out_size = mode, (out_size, out_size) if isinstance(out_size, int) else tuple(out_size)
    self.resize_min, self.resize_max, self.area, self.pad = int(resize_min), int(resize_max), tuple(area), int(pad)
    self.mean = tuple(mean) if mean is not None else (_VGG_MEANS if mode == "vgg" else (0.0, 0.0, 0.0))
    self.scale, self.seed = float(scale), int(seed)
    self._counters = {}   # device -> int64 step counter (device resident: graph-replayable augmentation)
    self.host_step = 0

  @property
  def stochastic(self):
    return self.mode in ("vgg", "inception", "cifarnet")

  def counter(self, device):
    device = torch.device(device)
    if device.type == "cuda" and device.index is None:
      device = torch.device("cuda", torch.cuda.current_device())
    if device not in self._counters:
      self._counters[device] = torch.zeros(1, dtype=torch.int64, device=device)
    return self._counters[device]

  def advance(self, device):
    """One-element device add (captured with the step under CUDA graphs, so every replay augments differently)."""
    self.counter(device).add_(1)
    self.host_step += 1

  # ------------------------------------------------------------------------------------------------ #
  def __call__(self, images, dtype, training, backend="torch", advance=True, stream_id=0, trigger=None):
    """`stream_id` decorrelates callers sharing this object (logical workers): it is folded into the seed. `trigger` = (groups, first,
    q): the backdoor trigger on the images `ops.nn.stamp_trigger` poisons (None: none)."""
    if images.dim() == 3:
      images = images[..., None]
    n, sh, sw, c = images.shape
    seed = (self.seed + 0x9E3779B1 * int(stream_id)) & _M64
    out = None
    if backend == "native" and images.is_cuda and images.dtype == torch.uint8 and c <= 3 and dtype in (torch.bfloat16, torch.float32):
      out = self._native(images.contiguous(), dtype, training, seed, trigger)
    if out is None:
      step = int(self.counter(images.device).item()) if training and self.stochastic else 0
      out = self._torch(images, dtype, training, step, seed, trigger)
    if training and self.stochastic and advance:
      self.advance(images.device)
    return out

  def _native(self, images, dtype, training, seed, trigger=None):
    from . import nn_native
    n, sh, sw, c = images.shape
    oh, ow = self.out_size
    out = torch.empty((n, oh, ow, c), dtype=dtype, device=images.device)
    ints = (ctypes.c_int * 12)(n, sh, sw, c, oh, ow, MODES[self.mode], 1 if training else 0, 1 if dtype == torch.float32 else 0, self.resize_min, self.resize_max, self.pad)
    floats = (ctypes.c_float * 6)(self.area[0], self.area[1], self.mean[0], self.mean[1], self.mean[2], self.scale)
    counter = self.counter(images.device)
    if trigger is not None:
      from .nn import trigger_descriptor
      rows, first, q, side = trigger_descriptor(out, trigger)
      nn_native._check(nn_native._lib().agb_image_preprocess_backdoor(nn_native._ptr(images), nn_native._ptr(out), ints, floats, ctypes.c_ulonglong(seed),
                                                                      nn_native._ptr(counter), ctypes.c_int(rows), ctypes.c_int(first), ctypes.c_int(q),
                                                                      ctypes.c_int(side), nn_native._stream()), "image_preprocess")
      return out.permute(0, 3, 1, 2)
    nn_native._check(nn_native._lib().agb_image_preprocess(nn_native._ptr(images), nn_native._ptr(out), ints, floats, ctypes.c_ulonglong(seed),
                                                           nn_native._ptr(counter), nn_native._stream()), "image_preprocess")
    return out.permute(0, 3, 1, 2)

  # -- the same arithmetic in numpy (parameters) + torch (pixels) ---------------------------------------- #
  def sampling(self, n, sh, sw, training, step, seed=None):
    """Per-image (y0, x0, sy, sx, flip, zero_outside) + colour parameters: numpy replica of `make_sampling`."""
    oh, ow = self.out_size
    idx = np.arange(n)
    seed = self.seed if seed is None else seed
    rnd = lambda slot: uniform01(seed, step, idx, slot)
    f32 = np.float32
    p = {"flip": np.zeros(n, dtype=bool), "zero_outside": False, "ordering": np.full(n, -1), "brightness": np.zeros(n, f32), "contrast": np.ones(n, f32),
         "saturation": np.ones(n, f32), "hue": np.zeros(n, f32)}
    if self.mode == "vgg":
      r = (self.resize_min + np.floor(rnd(0) * f32(self.resize_max - self.resize_min + 1))).astype(f32) if training else np.full(n, self.resize_min, f32)
      scale = r / f32(min(sh, sw))
      rh, rw = f32(sh) * scale, f32(sw) * scale
      oy = (rnd(1) if training else f32(0.5)) * np.maximum(rh - f32(oh), f32(0))
      ox = (rnd(2) if training else f32(0.5)) * np.maximum(rw - f32(ow), f32(0))
      p.update(y0=np.floor(oy) / scale, x0=np.floor(ox) / scale, sy=f32(1) / scale, sx=f32(1) / scale)
      if training:
        p["flip"] = rnd(3) < 0.5
    elif self.mode == "inception":
      bh, bw = np.full(n, sh, f32), np.full(n, sw, f32)
      if training:
        done = np.zeros(n, dtype=bool)
        for attempt in range(10):
          aspect = f32(0.75) + rnd(8 + 2 * attempt) * f32(4.0 / 3.0 - 0.75)
          area = (f32(self.area[0]) + rnd(9 + 2 * attempt) * f32(self.area[1] - self.area[0])) * f32(sh) * f32(sw)
          w, h = np.sqrt(area * aspect), np.sqrt(area / aspect)
          ok = (~done) & (w <= sw) & (h <= sh) & (w >= 1) & (h >= 1)
          bw, bh = np.where(ok, w, bw), np.where(ok, h, bh)
          done |= ok
        y0, x0 = rnd(1) * (f32(sh) - bh), rnd(2) * (f32(sw) - bw)
        p.update(flip=rnd(3) < 0.5, ordering=(rnd(4) * f32(4)).astype(np.int64) & 3, brightness=(f32(2) * rnd(5) - f32(1)) * f32(32.0 / 255.0),
                 saturation=f32(0.5) + rnd(6), hue=(f32(2) * rnd(7) - f32(1)) * f32(0.2), contrast=f32(0.5) + rnd(28))
      else:
        bh, bw = f32(0.875) * bh, f32(0.875) * bw
        y0, x0 = f32(0.5) * (f32(sh) - bh), f32(0.5) * (f32(sw) - bw)
      p.update(y0=y0, x0=x0, sy=bh / f32(oh), sx=bw / f32(ow))
    elif self.mode == "cifarnet":
      range_y, range_x = sh + 2 * self.pad - oh, sw + 2 * self.pad - ow
      oy = np.floor(rnd(1) * f32(range_y + 1)) if training else np.full(n, range_y // 2, f32)
      ox = np.floor(rnd(2) * f32(range_x + 1)) if training else np.full(n, range_x // 2, f32)
      p.update(y0=(oy - self.pad).astype(f32), x0=(ox - self.pad).astype(f32), sy=np.ones(n, f32), sx=np.ones(n, f32), zero_outside=True)
      if training:
        p.update(flip=rnd(3) < 0.5, brightness=(f32(2) * rnd(5) - f32(1)) * f32(63), contrast=f32(0.2) + rnd(6) * f32(1.6))
    else:
      p.update(y0=np.zeros(n, f32), x0=np.zeros(n, f32), sy=np.full(n, sh / oh, f32), sx=np.full(n, sw / ow, f32))
    return p

  def _torch(self, images, dtype, training, step, seed=None, trigger=None):
    n, sh, sw, c = images.shape
    oh, ow = self.out_size
    dev = images.device
    p = self.sampling(n, sh, sw, training, step, seed)
    t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float32), device=dev)
    flip = torch.as_tensor(np.asarray(p["flip"]), device=dev)
    xs = torch.arange(ow, device=dev, dtype=torch.float32)[None, :].expand(n, ow)
    xs = torch.where(flip[:, None], (ow - 1) - xs, xs)
    fy = t(p["y0"])[:, None] + torch.arange(oh, device=dev, dtype=torch.float32)[None, :] * t(p["sy"])[:, None]   # [n, oh]
    fx = t(p["x0"])[:, None] + xs * t(p["sx"])[:, None]                                                            # [n, ow]
    y0, x0 = torch.floor(fy), torch.floor(fx)
    wy, wx = (fy - y0)[:, :, None, None], (fx - x0)[:, None, :, None]
    src = images.to(torch.float32)
    batch = torch.arange(n, device=dev)[:, None, None]

    def gather(yi, xi):
      yi, xi = yi.long(), xi.long()
      if p["zero_outside"]:
        inside = ((yi >= 0) & (yi < sh))[:, :, None] & ((xi >= 0) & (xi < sw))[:, None, :]
        vals = src[batch, yi.clamp(0, sh - 1)[:, :, None], xi.clamp(0, sw - 1)[:, None, :]]
        return vals * inside[..., None]
      return src[batch, yi.clamp(0, sh - 1)[:, :, None], xi.clamp(0, sw - 1)[:, None, :]]

    v = ((1 - wy) * (1 - wx)) * gather(y0, x0) + ((1 - wy) * wx) * gather(y0, x0 + 1) + (wy * (1 - wx)) * gather(y0 + 1, x0) + (wy * wx) * gather(y0 + 1, x0 + 1)  # [n, oh, ow, c]
    if trigger is not None:
      from .nn import stamp_trigger
      v = stamp_trigger(v, *trigger)
    per = lambda a: t(a)[:, None, None, None]
    if self.mode == "inception":
      v = v / 255.0
      if training:
        order = np.asarray(p["ordering"])
        v = _colour_ops(v, p, order, c, True, per)
        mean = v.mean(dim=(1, 2), keepdim=True)
        v = (v - mean) * per(p["contrast"]) + mean
        v = _colour_ops(v, p, order, c, False, per)
        v = v.clamp(0.0, 1.0)
      v = (v - 0.5) * 2.0
    elif self.mode == "cifarnet":
      v = v + per(p["brightness"])
      mean = v.mean(dim=(1, 2), keepdim=True)
      v = (v - mean) * per(p["contrast"]) + mean
      # the variance around the mean of the channel means (what the contrast keeps), as the kernel takes it
      centre = mean.mean(dim=3, keepdim=True)
      d = v - centre
      shift = d.mean(dim=(1, 2, 3), keepdim=True)
      var = ((d * d).mean(dim=(1, 2, 3), keepdim=True) - shift * shift).clamp_min(0.0)
      v = (v - (centre + shift)) / torch.maximum(var.sqrt(), torch.full_like(var, 1.0 / math.sqrt(oh * ow * c)))
    else:
      v = (v - torch.tensor(self.mean[:c], device=dev, dtype=torch.float32)) * self.scale
    return v.to(dtype).permute(0, 3, 1, 2)


def _saturation(v, factor):
  gray = 0.2989 * v[..., 0:1] + 0.587 * v[..., 1:2] + 0.114 * v[..., 2:3]
  return gray + (v - gray) * factor


def _hue(v, delta):
  angle = 2.0 * math.pi * delta
  cs, sn = torch.cos(angle), torch.sin(angle)
  r, g, b = v[..., 0:1], v[..., 1:2], v[..., 2:3]
  y = 0.299 * r + 0.587 * g + 0.114 * b
  i = 0.596 * r - 0.274 * g - 0.322 * b
  q = 0.211 * r - 0.523 * g + 0.312 * b
  i2, q2 = i * cs - q * sn, i * sn + q * cs
  return torch.cat([y + 0.956 * i2 + 0.621 * q2, y - 0.272 * i2 - 0.647 * q2, y - 1.106 * i2 + 1.703 * q2], dim=-1)


def _colour_ops(v, p, order, channels, before, per):
  """slim `distort_color` operations before / after the contrast adjustment, per-image ordering (see `colour_ops` in the kernel)."""
  rgb = channels == 3
  out = v.clone()
  for o in range(4):
    rows = np.nonzero(order == o)[0]
    if len(rows) == 0:
      continue
    sel = torch.as_tensor(rows, device=v.device)
    x = v[sel]
    sub = lambda a: per(np.asarray(a)[rows])
    bright = lambda z: z + sub(p["brightness"])
    sat = (lambda z: _saturation(z, sub(p["saturation"]))) if rgb else (lambda z: z)
    hue = (lambda z: _hue(z, sub(p["hue"]))) if rgb else (lambda z: z)
    if o == 0 and before:
      x = hue(sat(bright(x)))
    elif o == 1:
      x = bright(sat(x)) if before else hue(x)
    elif o == 2 and not before:
      x = sat(bright(hue(x)))
    elif o == 3:
      x = sat(hue(x)) if before else bright(x)
    out[sel] = x
  return out

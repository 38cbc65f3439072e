"""Device preprocessing (`native/op_nn/preprocess.cu`) against a float64 oracle of its documented semantics.

The oracle draws the per-image random numbers with `ops.preprocess.uniform01` (values k / 2^24, exact in float64), derives the
crop, box, flip and colour parameters from them in float64, and samples, colours, adjusts contrast, clips and standardises in
float64. `test_oracle_matches_torch_float64` checks it against torch's float64 operators without a GPU.

Some parameters are discrete decisions (the floor of a crop offset, the acceptance of an Inception box, flip < 0.5, the colour
ordering) that fp32 arithmetic with contracted multiply-adds may take differently from float64 near their boundary. The oracle
reports the margin of each decision, and every case asserts that its seed and step counter leave each decision a margin far above
fp32 rounding, so the comparison is deterministic and no image or pixel is excluded.

Every pixel is then compared with a bound derived per image from: the fp32 error of the sampling coordinates times the largest
change (255) between neighbouring uint8 pixels; the colour chain, op by op; the per-image reductions (with the cancellation in
the contrast pivot and the standardisation variance); and the rounding of the output.
"""

import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from aggregathor_b200.ops.preprocess import Preprocessor, uniform01

F64 = torch.float64
U24 = 2.0 ** -24                        # unit roundoff of fp32
gpu = pytest.mark.gpu
GRAY = (0.2989, 0.587, 0.114)           # tf.image.rgb_to_grayscale
YIQ = np.array([[0.299, 0.587, 0.114], [0.596, -0.274, -0.322], [0.211, -0.523, 0.312]])
IYQ = np.array([[1.0, 0.956, 0.621], [1.0, -0.272, -0.647], [1.0, -1.106, 1.703]])


def _f32(x):
  return float(np.float32(x))


# ---------------------------------------------------------------------------- #
# float64 oracle

def _floor_margin(x):
  """Distance of x >= 0 from the nearest boundary its floor could cross (0 is no boundary: the operands are non-negative)."""
  f = math.floor(x)
  return f + 1 - x if f == 0 else min(x - f, f + 1 - x)


def sampling_ref(pre, n, sh, sw, training, step, seed):
  """Per-image parameters of `make_sampling`, in float64 from the kernel's uniforms:
    vgg        r = rmin + floor(u0 (rmax - rmin + 1)) (train) or rmin; scale = r / min(SH, SW); crop offset o = floor(u (R - O)) (train)
               or floor((R - O) / 2), R = S * scale; origin o / scale, step 1 / scale; flip u3 < 1/2 (train)
    inception  train: up to 10 boxes, aspect = 3/4 + u (4/3 - 3/4), area = (amin + u (amax - amin)) SH SW, w = sqrt(area aspect),
               h = sqrt(area / aspect), the first with w <= SW, h <= SH, w >= 1, h >= 1 (else the whole image); origin u (S - box);
               flip u3 < 1/2, ordering floor(4 u4), brightness (2 u5 - 1) 32/255, saturation 1/2 + u6, hue (2 u7 - 1) / 5,
               contrast 1/2 + u28; eval: the central 87.5 % box. Step = box / out.
    cifarnet   crop offset floor(u (S + 2 pad - O + 1)) (train) or (S + 2 pad - O) // 2, origin offset - pad, step 1, zero outside;
               train: flip, brightness (2 u5 - 1) 63, contrast 0.2 + 1.6 u6
    plain      origin 0, step S / O
  Returns a list of dicts, and the decisions as (name, image, margin, fp32 error scale of the decision variable)."""
  oh, ow = pre.out_size
  rnd = lambda slot: uniform01(seed, step, np.arange(n), slot).astype(np.float64)
  u = {slot: rnd(slot) for slot in list(range(29))}
  params, decisions = [], []
  for i in range(n):
    p = dict(flip=False, zero_outside=False, ordering=-1, brightness=0.0, contrast=1.0, saturation=1.0, hue=0.0, err_scale=0.0)
    if pre.mode == "vgg":
      if training:
        x = u[0][i] * (pre.resize_max - pre.resize_min + 1)
        decisions.append(("vgg size", i, _floor_margin(x), x))
        r = pre.resize_min + math.floor(x)
      else:
        r = pre.resize_min
      scale = r / min(sh, sw)
      offs = []
      for axis, (src, out) in enumerate(((sh, oh), (sw, ow))):
        o = (u[1 + axis][i] if training else 0.5) * max(src * scale - out, 0.0)
        decisions.append(("vgg offset", i, _floor_margin(o), src * scale))
        offs.append(math.floor(o) / scale)
      p.update(y0=offs[0], x0=offs[1], sy=1 / scale, sx=1 / scale, flip=training and u[3][i] < 0.5)
    elif pre.mode == "inception":
      bh, bw, y0, x0 = float(sh), float(sw), 0.0, 0.0
      if training:
        amin, amax = _f32(pre.area[0]), _f32(pre.area[1])
        for attempt in range(10):
          aspect = 0.75 + u[8 + 2 * attempt][i] * (_f32(4.0 / 3.0) - 0.75)
          area = (amin + u[9 + 2 * attempt][i] * (amax - amin)) * sh * sw
          w, h = math.sqrt(area * aspect), math.sqrt(area / aspect)
          slack = (sw - w, sh - h, w - 1, h - 1)
          ok = min(slack) >= 0
          decisions.append(("inception box", i, min(slack) if ok else max(-s for s in slack if s < 0), max(sh, sw, w, h)))
          if ok:
            bh, bw = h, w
            break
        y0, x0 = u[1][i] * (sh - bh), u[2][i] * (sw - bw)
        p.update(flip=u[3][i] < 0.5, ordering=int(math.floor(u[4][i] * 4)) & 3, brightness=(2 * u[5][i] - 1) * (32 / 255), saturation=0.5 + u[6][i],
                 hue=(2 * u[7][i] - 1) * 0.2, contrast=0.5 + u[28][i])
      else:
        bh, bw = 0.875 * sh, 0.875 * sw
        y0, x0 = 0.5 * (sh - bh), 0.5 * (sw - bw)
      p.update(y0=y0, x0=x0, sy=bh / oh, sx=bw / ow, err_scale=max(sh, sw))
    elif pre.mode == "cifarnet":
      offs = []
      for axis, (src, out) in enumerate(((sh, oh), (sw, ow))):
        rng = src + 2 * pre.pad - out
        if training:
          x = u[1 + axis][i] * (rng + 1)
          decisions.append(("cifarnet offset", i, _floor_margin(x), rng + 1))
          offs.append(math.floor(x) - pre.pad)
        else:
          offs.append(rng // 2 - pre.pad)
      p.update(y0=float(offs[0]), x0=float(offs[1]), sy=1.0, sx=1.0, zero_outside=True)
      if training:
        p.update(flip=u[3][i] < 0.5, brightness=(2 * u[5][i] - 1) * 63, contrast=0.2 + u[6][i] * _f32(1.6))
    else:
      p.update(y0=0.0, x0=0.0, sy=sh / oh, sx=sw / ow)
    params.append(p)
  return params, decisions


def bilinear_ref(img, p, oh, ow):
  """TF1 `resize_bilinear` sampling of the source box: pixel (oy, ox) reads fy = y0 + oy sy, fx = x0 + ox' sx (ox' = OW - 1 - ox when
  flipped), bilinear between the four neighbours; outside the image: 0 (zero_outside) or the nearest border pixel. img [SH, SW, C]."""
  sh, sw, c = img.shape
  src = img.astype(np.float64)
  oxs = np.arange(ow)
  if p["flip"]:
    oxs = ow - 1 - oxs
  fy, fx = p["y0"] + np.arange(oh) * p["sy"], p["x0"] + oxs * p["sx"]
  y0, x0 = np.floor(fy), np.floor(fx)
  wy, wx = (fy - y0)[:, None, None], (fx - x0)[None, :, None]
  out = np.zeros((oh, ow, c))
  for dy in (0, 1):
    for dx in (0, 1):
      y, x = (y0 + dy).astype(np.int64), (x0 + dx).astype(np.int64)
      if p["zero_outside"]:
        vals = src[np.clip(y, 0, sh - 1)][:, np.clip(x, 0, sw - 1)] * (((y >= 0) & (y < sh))[:, None, None] & ((x >= 0) & (x < sw))[None, :, None])
      else:
        vals = src[np.clip(y, 0, sh - 1)][:, np.clip(x, 0, sw - 1)]
      out += (wy if dy else 1 - wy) * (wx if dx else 1 - wx) * vals
  return out


def saturation_ref(v, f):
  gray = v @ np.array(GRAY)
  return gray[..., None] + (v - gray[..., None]) * f


def hue_matrix(delta):
  """Rotation of the YIQ chroma plane by `delta` turns, as one 3 x 3 matrix on RGB."""
  cs, sn = math.cos(2 * math.pi * delta), math.sin(2 * math.pi * delta)
  rot = np.array([[1.0, 0.0, 0.0], [0.0, cs, -sn], [0.0, sn, cs]])
  return IYQ @ rot @ YIQ


def colour_ref(v, p, channels, before):
  """slim `distort_color` orderings (0 = B S H C, 1 = S B C H, 2 = C H B S, 3 = H S C B), the part before or after the contrast."""
  rgb = channels == 3
  ops = {"B": lambda z: z + p["brightness"], "S": (lambda z: saturation_ref(z, p["saturation"])) if rgb else (lambda z: z),
         "H": (lambda z: z @ hue_matrix(p["hue"]).T) if rgb else (lambda z: z)}
  seq = ["BSHC", "SBCH", "CHBS", "HSCB"][p["ordering"]]
  part = seq[:seq.index("C")] if before else seq[seq.index("C") + 1:]
  for op in part:
    v = ops[op](v)
  return v, part


def preprocess_ref(pre, images, training, step, seed):
  """uint8 [N, SH, SW, C] -> float64 [N, OH, OW, C] and the per-image parameters:
    inception  v / 255, colour ops before the contrast (train), contrast (v - mean_c) f + mean_c with the per-channel image mean,
               colour ops after, clip to [0, 1] (train); then (v - 1/2) 2
    cifarnet   v + brightness, contrast around mean_c (train), then per-image standardisation over all values:
               (v - m) / max(std, 1 / sqrt(OH OW C)) with the biased std
    vgg/plain  (v - mean[c]) * scale"""
  n, sh, sw, c = images.shape
  oh, ow = pre.out_size
  params, decisions = sampling_ref(pre, n, sh, sw, training, step, seed)
  out = np.zeros((n, oh, ow, c))
  for i in range(n):
    p = params[i]
    v = bilinear_ref(images[i], p, oh, ow)
    p["sample"] = v
    if pre.mode == "inception":
      v = v / 255
      if training:
        v, _ = colour_ref(v, p, c, True)
        p["before"] = v
        mean = v.mean(axis=(0, 1))
        v = (v - mean) * p["contrast"] + mean
        p["contrasted"] = v
        v, _ = colour_ref(v, p, c, False)
        p["after"] = v
        v = np.clip(v, 0.0, 1.0)
      v = (v - 0.5) * 2
    elif pre.mode == "cifarnet":
      v = v + p["brightness"]
      p["bright"] = v
      mean = v.mean(axis=(0, 1))
      v = (v - mean) * p["contrast"] + mean
      p["contrasted"] = v
      m = v.mean()
      std = math.sqrt(((v - m) ** 2).mean())
      p.update(m=m, std=std, floor=1 / math.sqrt(v.size))
      v = (v - m) / max(std, p["floor"])
    else:
      v = (v - np.array([_f32(x) for x in pre.mean[:c]])) * _f32(pre.scale)
    out[i] = v
  return out, params, decisions


# ---------------------------------------------------------------------------- #
# Oracle self-check (no GPU)

def _hash_uniform(seed, step, image, slot):
  """`uniform01` with Python integers."""
  m = (1 << 64) - 1
  h = (seed ^ (step * 0x9E3779B97F4A7C15 & m) ^ (((image << 32) | slot) * 0xD1B54A32D192ED03 & m)) & m
  for mul in (0xff51afd7ed558ccd, 0xc4ceb9fe1a85ec53):
    h ^= h >> 33
    h = h * mul & m
  h ^= h >> 33
  return (h >> 40) / 2.0 ** 24


def test_oracle_matches_torch_float64():
  rng = np.random.default_rng(0)
  for seed, step in ((11, 7), (3, 1 << 41), ((1 << 64) - 5, (1 << 63) + 9)):
    got = uniform01(seed, step, np.arange(5), 28)
    assert [float(g) for g in got] == [_hash_uniform(seed, step, i, 28) for i in range(5)]
  # bilinear sampling vs grid_sample (align_corners: normalised -1 / +1 are the centres of the first / last pixels)
  img = rng.integers(0, 256, (13, 17, 3), dtype=np.uint8)
  for p in (dict(y0=-1.25, x0=2.5, sy=0.7, sx=1.3, flip=True, zero_outside=False), dict(y0=-2.0, x0=3.0, sy=1.0, sx=1.0, flip=False, zero_outside=True),
            dict(y0=0.3, x0=-0.6, sy=1.9, sx=0.45, flip=False, zero_outside=True)):
    oh, ow = 9, 11
    want_src = torch.from_numpy(img).to(F64).permute(2, 0, 1)[None]
    oxs = np.arange(ow)[::-1] if p["flip"] else np.arange(ow)
    fy, fx = p["y0"] + np.arange(oh) * p["sy"], p["x0"] + oxs * p["sx"]
    gy = torch.from_numpy(2 * fy / (13 - 1) - 1)[:, None].expand(oh, ow)
    gx = torch.from_numpy(2 * fx / (17 - 1) - 1)[None, :].expand(oh, ow)
    grid = torch.stack([gx, gy], dim=-1)[None]
    want = F.grid_sample(want_src, grid, mode="bilinear", padding_mode="zeros" if p["zero_outside"] else "border", align_corners=True)[0].permute(1, 2, 0)
    torch.testing.assert_close(torch.from_numpy(bilinear_ref(img, p, oh, ow)), want, rtol=1e-12, atol=1e-9)
  # colour operations: saturation interpolates from the gray level, the hue matrix keeps Y and the length of (I, Q) and rotates it
  # by 2 pi delta
  v = torch.from_numpy(rng.random((7, 3)))
  s = torch.from_numpy(saturation_ref(v.numpy(), 1.3))
  gray = (v @ torch.tensor(GRAY, dtype=F64))[:, None].expand(7, 3)
  torch.testing.assert_close(s, torch.lerp(gray, v, 1.3), rtol=1e-12, atol=1e-12)
  yiq = torch.from_numpy(YIQ)
  iyq = torch.linalg.inv(yiq)
  torch.testing.assert_close(iyq, torch.from_numpy(IYQ), rtol=0, atol=3e-3)   # the kernel's rounded inverse of YIQ
  h = torch.from_numpy(v.numpy() @ hue_matrix(0.15).T)
  a, b = v @ yiq.T, h @ torch.linalg.inv(torch.from_numpy(IYQ)).T
  torch.testing.assert_close(b[:, 0], a[:, 0], rtol=1e-12, atol=1e-12)
  ang = torch.remainder(torch.atan2(b[:, 2], b[:, 1]) - torch.atan2(a[:, 2], a[:, 1]), 2 * math.pi)
  torch.testing.assert_close(ang, torch.full((7,), 0.3 * math.pi, dtype=F64), rtol=0, atol=1e-9)
  torch.testing.assert_close(torch.linalg.vector_norm(b[:, 1:], dim=1), torch.linalg.vector_norm(a[:, 1:], dim=1), rtol=1e-12, atol=1e-12)
  # cifarnet: contrast keeps the channel means, standardisation = torch's mean / biased std, floored
  pre = Preprocessor("cifarnet", 8, pad=0, seed=5)
  images = rng.integers(0, 256, (3, 8, 8, 3), dtype=np.uint8)
  images[2] = 9
  out, params, _ = preprocess_ref(pre, images, True, 4, 5)
  for i in range(3):
    t = torch.from_numpy(params[i]["contrasted"])
    torch.testing.assert_close(t.mean(dim=(0, 1)), torch.from_numpy(params[i]["bright"]).mean(dim=(0, 1)), rtol=1e-12, atol=1e-9)
    std = torch.maximum(t.std(unbiased=False), torch.tensor(1 / math.sqrt(t.numel()), dtype=F64))
    torch.testing.assert_close(torch.from_numpy(out[i]), (t - t.mean()) / std, rtol=1e-12, atol=1e-9)
  assert float(np.abs(out[2]).max()) < 1e-9 and params[2]["std"] < params[2]["floor"]   # a uniform image sits on the floor
  # inception eval: the central 87.5 % box resized, then [-1, 1]
  pre = Preprocessor("inception", (6, 5))
  out, params, _ = preprocess_ref(pre, images, False, 0, 0)
  src = torch.from_numpy(images).to(F64).permute(0, 3, 1, 2)
  gy = torch.from_numpy((0.0625 * 8 + np.arange(6) * 7 / 6) * 2 / 7 - 1)[:, None].expand(6, 5)
  gx = torch.from_numpy((0.0625 * 8 + np.arange(5) * 7 / 5) * 2 / 7 - 1)[None, :].expand(6, 5)
  want = F.grid_sample(src, torch.stack([gx, gy], dim=-1)[None].expand(3, 6, 5, 2), mode="bilinear", padding_mode="border", align_corners=True)
  torch.testing.assert_close(torch.from_numpy(out), (want / 255 - 0.5).permute(0, 2, 3, 1) * 2, rtol=1e-12, atol=1e-12)


# ---------------------------------------------------------------------------- #
# Bound

def _chain(pixels):
  """Longest fp32 addition chain behind a per-image sum: the strided per-thread partial (512 threads), the warp shuffle (5),
  the fold over 16 warps, then the division."""
  return -(-pixels // 512) + 5 + 16 + 1


def _ulp(ref, bf16):
  mant = 7 if bf16 else 23
  _, e = np.frexp(np.maximum(np.abs(ref), 2.0 ** -126))
  return np.ldexp(1.0, e - 1 - mant)


def _op_norm(part, p):
  """(infinity norm of the linear colour map, of its absolute coefficients) of the ops in `part` (B, S, H)."""
  norm, absn = np.eye(3), np.eye(3)
  for op in part:
    if op == "S":
      m = np.eye(3) * p["saturation"] + (1 - p["saturation"]) * np.ones((3, 1)) @ np.array(GRAY)[None]
      a = np.eye(3) * abs(p["saturation"]) + abs(1 - p["saturation"]) * np.ones((3, 1)) @ np.array(GRAY)[None] + np.ones((3, 1)) @ np.array(GRAY)[None]
    elif op == "H":
      cs, sn = math.cos(2 * math.pi * p["hue"]), math.sin(2 * math.pi * p["hue"])
      m = hue_matrix(p["hue"])
      a = np.abs(IYQ) @ np.array([[1.0, 0, 0], [0, abs(cs), abs(sn)], [0, abs(sn), abs(cs)]]) @ np.abs(YIQ)
    else:
      continue
    norm, absn = m @ norm, a @ absn
  return np.abs(norm).sum(axis=1).max(), np.abs(absn).sum(axis=1).max()


def _colour_err(e, mag, part, p):
  """Error after the colour ops `part`, from an input error e on values of magnitude <= mag (0..1 scale): the map's norm carries e;
  brightness adds one rounding of the sum (and its own 3 of the parameter), saturation and hue round every product and sum
  (at most 12 per output, relative to the absolute-coefficient map, sincospif within 2 ulp on cos / sin)."""
  for op in part:
    a, absn = _op_norm(op, p)
    if op == "B":
      mag = mag + abs(p["brightness"])
      e = e + U24 * mag + 3 * U24 * abs(p["brightness"])
    else:
      e = a * e + 12 * U24 * absn * mag
      mag = absn * mag
  return e, mag


def image_bound(pre, p, images_i, training, bf16, ref):
  """Per-pixel bound for one image (see the module docstring); `ref` is the oracle's output for it."""
  sh, sw, c = images_i.shape
  oh, ow = pre.out_size
  if p["zero_outside"]:
    e = 0.0              # cifarnet: integer origins (< 2^24) and unit steps: fy = y0 + oy is exact, the weights are 0 / 1
  else:
    # coordinates: vgg's origin floor(o) / scale and step 1 / scale carry 2 u each (scale = r / S rounds once), plain's step S / O
    # one u, and fy = origin + index * step one more: 4 u of (|origin| + index * step) per axis. Inception's box adds the roundings
    # of its area, aspect, square roots and S - box difference, all of quantities up to the source size: 16 u of it (`err_scale`).
    # The bilinear value moves at most 255 per pixel of coordinate along each axis; the weights and the 4-tap sum round 8 times
    # values <= 255
    ey = 4 * U24 * (abs(p["y0"]) + oh * p["sy"]) + 16 * U24 * p["err_scale"]
    ex = 4 * U24 * (abs(p["x0"]) + ow * p["sx"]) + 16 * U24 * p["err_scale"]
    e = 255 * (ey + ex) + 8 * U24 * 255
  if pre.mode in ("vgg", "plain"):
    # (v - mean) * scale: mean and scale are the fp32 values; the difference and the product round once each
    return (e + 2 * U24 * (255 + abs(_f32(pre.mean[0])) + 256)) * abs(_f32(pre.scale)) + 2 * U24 * np.abs(ref) + _ulp(ref, bf16)
  if pre.mode == "inception":
    e = e / 255 + U24      # the 1 / 255 product (the constant and the product round)
    mag = 1.0
    if training:
      ordering = "BSHC", "SBCH", "CHBS", "HSCB"
      seq = ordering[p["ordering"]]
      before, after = seq[:seq.index("C")], seq[seq.index("C") + 1:]
      if c == 1:
        before, after = before.replace("S", "").replace("H", ""), after.replace("S", "").replace("H", "")
      e, mag = _colour_err(e, mag, before, p)
      mag = max(mag, float(np.abs(p["before"]).max()))
      # contrast (v - m) f + m with m the fp32 per-channel mean: e plus a chain of additions of values <= mag; f = 1/2 + u28
      # (one rounding); three roundings of values <= (1 + f) mag
      em = e + _chain(oh * ow) * U24 * mag
      f = p["contrast"]
      e = f * (e + em) + em + U24 * f * 2 * mag + 3 * U24 * (1 + f) * 2 * mag
      mag = max(mag, float(np.abs(p["contrasted"]).max()))
      e, mag = _colour_err(e, mag, after, p)
      # the clip is 1-Lipschitz
    return 2 * e + 2 * U24 * 2 + _ulp(ref, bf16)
  # cifarnet
  bright = p["bright"]
  m1 = float(np.abs(bright).max())
  e1 = U24 * (63 * 1 + m1)                     # brightness = (2 u5 - 1) * 63 rounds once, the sum once
  emc = e1 + _chain(oh * ow) * U24 * m1        # per-channel mean
  f = p["contrast"]
  d1 = float(np.abs(bright - bright.mean(axis=(0, 1))).max())
  e2 = f * e1 + (1 + f) * emc + 3 * U24 * f * d1 + 4 * U24 * (m1 + f * d1)   # (v - m_c) f + m_c, f = 0.2 + 1.6 u6 with 3 roundings
  v2 = p["contrasted"]
  n = v2.size
  # standardisation: the sums run over d = v - p with p the mean of the channel means (within e_p of its float64 value), in chains of
  # L2 additions; the mean is p + t0 / N, the variance t1 / N - (t0 / N)^2
  ep = emc + 2 * U24 * m1
  L2 = _chain(oh * ow * c)
  d = v2 - v2.mean() + (v2.mean(axis=(0, 1)).mean() - v2.mean())    # the float64 d around the oracle's pivot
  ed = e2 + ep + U24 * np.abs(d)
  t0e = float(ed.sum() + L2 * U24 * np.abs(d).sum())
  t1e = float((2 * np.abs(d) * ed + ed ** 2).sum() + (L2 + 1) * U24 * (d * d).sum())
  md = float(d.mean())
  e_var = t1e / n + 2 * abs(md) * t0e / n + (t0e / n) ** 2 + 3 * U24 * (float((d * d).mean()) + md * md)
  sf = max(p["std"], p["floor"])
  rel = e_var / sf / sf + 4 * U24              # |sqrt a - sqrt b| <= |a - b| / sf, max() is 1-Lipschitz; sqrt, rsqrtf, 1 / x
  em = ep + t0e / n + U24 * abs(p["m"])
  return (e2 + em + U24 * np.abs(v2 - p["m"])) / sf + np.abs(ref) * (rel + U24) + _ulp(ref, bf16)


# ---------------------------------------------------------------------------- #
# Native runs

class _Recorder:
  """Stands in for the native library: forwards everything, records the status of every preprocessing launch."""

  def __init__(self, lib):
    self._lib = lib
    self.calls = []

  def __getattr__(self, name):
    fn = getattr(self._lib, name)
    if not name.startswith("agb_image_preprocess"):
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


def _random_images(n, sh, sw, c, seed):
  return np.random.default_rng(seed).integers(0, 256, (n, sh, sw, c), dtype=np.uint8)


def run_case(record, pre, images, training, step, dtype, what, min_margin=1.0):
  """One native launch at step counter `step` against the oracle; every decision margin at least `min_margin` times its fp32 error
  scale (64 u of the decision variable's operands)."""
  ref, params, decisions = preprocess_ref(pre, images, training, step, pre.seed)
  for name, image, margin, scale in decisions:
    need = 64 * U24 * max(scale, 1.0)
    assert margin >= min_margin * need, "%s: %s of image %d is %.3g from its boundary (needs %.3g): choose another seed" % (what, name, image, margin, need)
  x = torch.from_numpy(images).cuda()
  counter = pre.counter("cuda")
  counter.fill_(step)
  before = len(record.calls)
  out = pre(x, dtype, training, backend="native", advance=False)
  torch.cuda.synchronize()
  assert record.calls[before:] == [("agb_image_preprocess", 0)], (what, record.calls[before:])
  got = out.permute(0, 2, 3, 1).to(F64).cpu().numpy()
  assert got.shape == ref.shape
  bf16 = dtype == torch.bfloat16
  for i, p in enumerate(params):
    bound = image_bound(pre, p, images[i], training, bf16, ref[i])
    where = "%s image %d (flip=%d ordering=%d)" % (what, i, p["flip"], p["ordering"])
    if p["flip"]:                # the mirrored border first, so that a defect confined to it is named as such
      _check(got[i, :, -1], ref[i, :, -1], bound[:, -1] if np.ndim(bound) else bound, where + " last column")
      _check(got[i, -1], ref[i, -1], bound[-1] if np.ndim(bound) else bound, where + " last row")
    _check(got[i], ref[i], bound, where)
  return ref, params


def _check(got, ref, bound, what):
  bound = np.broadcast_to(bound, ref.shape)
  assert np.isfinite(got).all(), what + ": non-finite output"
  err = np.abs(got - ref)
  bad = err > bound
  if bad.any():
    first = tuple(np.argwhere(bad)[0])
    raise AssertionError("%s: %d of %d values out of bound; first at %s: got %r, oracle %r, bound %.3g (max err/bound %.3g)"
                         % (what, int(bad.sum()), bad.size, first, float(got[first]), float(ref[first]), float(bound[first]), float((err / bound).max())))


DTYPES = pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])


@gpu
@DTYPES
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("source", [(300, 257), (257, 420)], ids=["portrait", "landscape"])
def test_vgg(record, dtype, training, source):
  """Aspect-preserving resize to a short side in [256, 300] then a crop; vgg takes min(SH, SW), so portrait and landscape sources
  scale by their width and their height. Output 223 (an odd r - O: the central offset is half an integer)."""
  pre = Preprocessor("vgg", 223, resize_min=256, resize_max=300, seed=21)
  images = _random_images(6, *source, 3, 22)
  run_case(record, pre, images, training, 7, dtype, "vgg %s %s" % (source, "train" if training else "eval"))


@gpu
@DTYPES
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("channels", [3, 1])
def test_inception(record, dtype, training, channels):
  """Distorted boxes, mirror and every colour ordering (3 channels; brightness and contrast only with 1), and the central 87.5 %
  box; landscape source, 33 x 33 output (not a multiple of the 512 threads)."""
  pre = Preprocessor("inception", 33, seed=31)
  images = _random_images(16, 120, 150, channels, 32)
  _, params = run_case(record, pre, images, training, 5, dtype, "inception C=%d %s" % (channels, "train" if training else "eval"))
  if training:
    assert {p["ordering"] for p in params} == {0, 1, 2, 3} and {p["flip"] for p in params} == {False, True}


@gpu
@DTYPES
def test_inception_every_box_rejected(record, dtype):
  """Area fractions in [0.9, 1] of a 100 x 160 source: every one of the 10 boxes needs an aspect above 4/3, all are rejected and
  the whole image is resized."""
  pre = Preprocessor("inception", (29, 31), area=(0.9, 1.0), seed=41)
  images = _random_images(6, 100, 160, 3, 42)
  ref, params, decisions = preprocess_ref(pre, images, True, 3, pre.seed)
  assert len(decisions) == 60 and all(p["sy"] == 100 / 29 and p["y0"] == 0.0 for p in params)
  run_case(record, pre, images, True, 3, dtype, "inception all boxes rejected")


@gpu
@DTYPES
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("channels", [3, 1])
def test_cifarnet(record, dtype, training, channels):
  """Pad 4 and a random 32 x 32 crop of a 36 x 30 source (zero rows and columns enter the window), mirror, brightness, contrast,
  per-image standardisation; and a 7 x 7 output (49 pixels, fewer than the 512 threads)."""
  for size, source, seed in ((32, (36, 30), 51), (7, (9, 8), 52)):
    pre = Preprocessor("cifarnet", size, pad=4, seed=seed)
    images = _random_images(8, *source, channels, seed + 100)
    run_case(record, pre, images, training, 11, dtype, "cifarnet %d C=%d %s" % (size, channels, "train" if training else "eval"))


@gpu
@DTYPES
def test_cifarnet_pad0_uniform_images(record, dtype):
  """Pad 0 and a source as large as the output (the only crop is the image itself); uniform images have zero variance and are
  standardised with the 1 / sqrt(N) floor."""
  pre = Preprocessor("cifarnet", 32, pad=0, seed=61)
  images = _random_images(6, 32, 32, 3, 62)
  images[1] = 0
  images[2] = 255
  images[3] = 77
  ref, params = run_case(record, pre, images, True, 2, dtype, "cifarnet pad 0 uniform")
  assert all(params[i]["std"] < params[i]["floor"] for i in (1, 2, 3))
  run_case(record, pre, images, False, 0, dtype, "cifarnet pad 0 uniform eval")


@gpu
@pytest.mark.parametrize("size", [32, 64])
def test_cifarnet_bright_nearly_uniform(record, size):
  """Values 250 +- 1, brightness above +40 and contrast near 0.2: the standardisation variance is about 0.02 on values of about
  300, so a variance formed as E[v^2] - E[v]^2 in fp32 loses most of its digits. Seeds chosen for strong brightness and weak contrast."""
  pre = Preprocessor("cifarnet", size, pad=0, seed=71)
  n = 16
  images = np.random.default_rng(72).integers(249, 252, (n, size, size, 3), dtype=np.uint8)
  step = _bright_step(pre, n)
  ref, params = run_case(record, pre, images, True, step, torch.float32, "cifarnet bright %d" % size)
  assert sum(p["brightness"] > 40 and p["contrast"] < 0.4 for p in params) >= 2


def _bright_step(pre, n):
  """The first step counter at which at least two of the n images draw brightness > 40 and contrast < 0.4."""
  for step in range(1000):
    b = (2 * uniform01(pre.seed, step, np.arange(n), 5).astype(np.float64) - 1) * 63
    f = 0.2 + uniform01(pre.seed, step, np.arange(n), 6).astype(np.float64) * 1.6
    if ((b > 40) & (f < 0.4)).sum() >= 2:
      return step
  raise AssertionError("no such step")


@gpu
@pytest.mark.parametrize("mode", ["vgg", "inception", "cifarnet"])
def test_large_step_counter(record, mode):
  """A step counter above 2^40: the hash takes the whole 64-bit counter (a 32-bit truncation would draw other parameters)."""
  step = (1 << 40) + 12345
  pre = Preprocessor(mode, 24, resize_min=30, resize_max=40, seed=81)
  images = _random_images(8, 40, 44, 3, 82)
  _, params, _ = preprocess_ref(pre, images, True, step, pre.seed)
  _, low, _ = preprocess_ref(pre, images, True, step & 0xFFFFFFFF, pre.seed)
  assert any(a["flip"] != b["flip"] or a["y0"] != b["y0"] for a, b in zip(params, low))
  run_case(record, pre, images, True, step, torch.float32, "%s step 2^40" % mode)


@gpu
@DTYPES
@pytest.mark.parametrize("channels", [1, 3])
def test_plain(record, dtype, channels):
  """(v - mean) * scale after a bilinear resize of the whole image, upsampling one axis and downsampling the other."""
  pre = Preprocessor("plain", (7, 40), mean=(128.0, 120.0, 100.0), scale=1 / 128.0)
  images = _random_images(5, 19, 23, channels, 91)
  run_case(record, pre, images, False, 0, dtype, "plain C=%d" % channels)

#!/usr/bin/env python3
"""GEMM / implicit-convolution products of the headline step (slim ResNet-50 v1, n = 8 batched logical workers x 32 images,
224x224, bf16): per-product kernel times with the staged and the register epilogue, and a kernel-time profile of the whole step.

    python benchmarks/nn_bench.py --dry-run                # product table with FLOP and byte counts (no GPU needed)
    python benchmarks/nn_bench.py --out DIR                # time every product, staged vs register epilogue alternating in one process
    python benchmarks/nn_bench.py --profile --out DIR      # torch.profiler pass over the headline step (run it on its own)
    python benchmarks/nn_bench.py --traffic                # HBM bytes of the batch-norm and residual passes (no GPU needed)

The products are derived from the model: a CPU forward pass at batch 1 records every Conv2d / Dense input shape, and the same
dispatch rules as `ops/nn_native.py` (1x1 stride-1 -> GEMM, implicit-GEMM conv, im2col + GEMM) turn each layer into its
forward, data-gradient and (grouped, split-K) weight-gradient products at the batched size. Results go to DIR/*.json.
"""

import argparse
import collections
import json
import math
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

SM_COUNT = 132   # H100 SXM: the split-K choice of the nn wrappers depends on it; the GPU run reads the real count


def parse():
  parser = argparse.ArgumentParser()
  parser.add_argument("--dry-run", action="store_true")
  parser.add_argument("--traffic", action="store_true")
  parser.add_argument("--profile", action="store_true")
  parser.add_argument("--out", type=str, default="nn_bench_out")
  parser.add_argument("--workers", type=int, default=8)
  parser.add_argument("--batch-size", type=int, default=32, help="per logical worker")
  parser.add_argument("--image-size", type=int, default=224)
  parser.add_argument("--seconds", type=float, default=0.25, help="length of one timing window (two per epilogue and product)")
  parser.add_argument("--steps", type=int, default=5, help="--profile: profiled steps")
  return parser.parse_args()


def card():
  """Name, power limit and SM clocks of GPU 0, read next to the numbers they qualify."""
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    return dict(zip(("name", "power_limit", "max_sm_clock", "sm_clock"), (s.strip() for s in out.split(","))))
  except (OSError, subprocess.SubprocessError):
    return {"name": torch.cuda.get_device_name(0) if torch.cuda.is_available() else None}


# ---------------------------------------------------------------------------- #
# Layer walk

def layer_shapes(image_size):
  """[(kind, layer, input shape (1, C, H, W) or (1, F), pads)] of every Conv2d / Dense of ResNet-50, in forward order."""
  from aggregathor_b200.engine.flat import FlatLayout
  from aggregathor_b200.models import Context, get_network
  from aggregathor_b200.models import core
  model = get_network("resnet_v1_50", 1000)
  layout, states = FlatLayout(), {}
  model.declare(layout, states)
  layout.freeze()
  params = torch.zeros(layout.padded_size)
  state = {k: torch.zeros(v) for k, v in states.items()}
  model.initialize(layout.views(params), state, torch.Generator().manual_seed(0))
  ctx = Context("torch", False, torch.float32, "cpu")
  ctx.master = ctx.weights = layout.views(params)
  ctx.state = state
  seen = []
  conv_forward, dense_forward = core.Conv2d.forward, core.Dense.forward

  def conv(self, x, c):
    seen.append(("conv", self, tuple(x.shape), self._pads(x.shape[2], x.shape[3])))
    return conv_forward(self, x, c)

  def dense(self, x, c):
    seen.append(("dense", self, (x.shape[0], x[0].numel()), None))
    return dense_forward(self, x, c)

  core.Conv2d.forward, core.Dense.forward = conv, dense
  try:
    x = torch.zeros((1, 3, image_size, image_size)).contiguous(memory_format=torch.channels_last)
    with torch.no_grad():
      model.root.forward(x, ctx)
  finally:
    core.Conv2d.forward, core.Dense.forward = conv_forward, dense_forward
  return seen


def _splits_tn(m, n, k, groups, deterministic):
  """`nn_native.mm_tn`'s split-K choice."""
  if deterministic:
    return 1
  bn = 64 if n <= 64 else 128
  tiles = ((m + 127) // 128) * ((n + bn - 1) // bn)
  want = max(1, (2 * SM_COUNT + tiles - 1) // tiles)
  return max(1, min((k + 63) // 64, want, 128) // groups)


def _splits_conv_wgrad(n, oh, ow, cin, cout, k, groups, deterministic):
  """`nn_native.conv2d_backward_implicit`'s split-K choice."""
  if deterministic:
    return 1
  tiles = k * k * ((cout + 127) // 128) * ((cin + 127) // 128)
  kblocks = max(1, n * oh * ow // 64 // groups)
  return max(1, min(kblocks, (2 * SM_COUNT + tiles * groups - 1) // (tiles * groups), 64))


def products(workers, batch, image_size, deterministic=False):
  """Distinct products of one step with their call counts. Each: dict(kind = gemm | conv, mode, shapes, flop, bytes, calls, layers)."""
  B = workers * batch
  table = collections.OrderedDict()

  def add(key, layer, **spec):
    if key not in table:
      table[key] = dict(spec, calls=0, layers=[])
    table[key]["calls"] += 1
    table[key]["layers"].append(layer)

  def gemm(layer, mode, M, N, K, a_mn, b_mn, out_fp32, groups=1, splits=1, bias=False):
    # bytes: operands read once and the output written once (split-K: one fp32 read-modify-write per split, counted as a write)
    flop = 2 * M * N * K * groups
    nbytes = 2 * (M * K + N * K) * groups + (4 if out_fp32 else 2) * M * N * groups * splits
    add(("gemm", mode, M, N, K, a_mn, b_mn, out_fp32, groups, splits, bias), layer, kind="gemm", mode=mode, M=M, N=N, K=K, a_mn=a_mn, b_mn=b_mn,
        out_fp32=out_fp32, groups=groups, splits=splits, bias=bias, flop=flop, bytes=nbytes)

  def conv(layer, mode, n, h, w, oh, ow, cin, cout, k, stride, pads, groups=1, splits=1):
    flop = 2 * n * oh * ow * cout * cin * k * k
    x_bytes, y_bytes, w_bytes = 2 * n * h * w * cin, 2 * n * oh * ow * cout, 2 * cout * k * k * cin
    nbytes = {0: x_bytes + w_bytes + y_bytes, 1: y_bytes + w_bytes + x_bytes, 2: x_bytes + y_bytes + 2 * w_bytes * groups * splits}[mode]
    add(("conv", mode, n, h, w, oh, ow, cin, cout, k, stride, tuple(pads), groups, splits), layer, kind="conv", mode=("fwd", "dgrad", "wgrad")[mode], n=n, h=h, w=w,
        oh=oh, ow=ow, cin=cin, cout=cout, k=k, stride=stride, pads=list(pads), groups=groups, splits=splits, flop=flop, bytes=nbytes)

  for kind, layer, shape, pads in layer_shapes(image_size):
    first = getattr(layer, "is_first", False)
    if kind == "dense":
      fin, fout = shape[1], layer.fout
      gemm(layer.name, "fwd", B, fout, fin, 0, 0, 0, bias=layer.bias)
      gemm(layer.name, "wgrad", fout, fin, B // workers, 1, 1, 1, workers, _splits_tn(fout, fin, B // workers, workers, deterministic))
      if not first:
        gemm(layer.name, "dgrad", B, fin, fout, 0, 1, 0)
      continue
    _, cin, h, w = shape
    cout, kh, kw, stride = layer.cout, layer.kh, layer.kw, layer.stride
    oh, ow = (h + pads[0] + pads[1] - kh) // stride + 1, (w + pads[2] + pads[3] - kw) // stride + 1
    if kh == kw == 1 and stride == 1 and not any(pads) and cin % 8 == 0:
      M = B * h * w
      gemm(layer.name, "fwd", M, cout, cin, 0, 0, 0, bias=layer.bias)
      gemm(layer.name, "wgrad", cout, cin, M // workers, 1, 1, 1, workers, _splits_tn(cout, cin, M // workers, workers, deterministic))
      if not first:
        gemm(layer.name, "dgrad", M, cin, cout, 0, 1, 0)
      continue
    implicit = kh == kw and kh > 1 and cin % 64 == 0 and cout % 64 == 0 and (
      (stride == 1 and kh % 2 == 1 and tuple(pads) == ((kh - 1) // 2,) * 4) or
      (stride == 2 and h % 2 == 0 and w % 2 == 0 and (oh, ow) == (h // 2, w // 2) and pads[0] < kh and pads[2] < kh))
    if implicit:
      conv(layer.name, 0, B, h, w, oh, ow, cin, cout, kh, stride, pads)
      conv(layer.name, 2, B, h, w, oh, ow, cin, cout, kh, stride, pads, workers, _splits_conv_wgrad(B, oh, ow, cin, cout, kh, workers, deterministic))
      if not first:
        conv(layer.name, 1, B, h, w, oh, ow, cin, cout, kh, stride, pads)
      continue
    kcol = kh * kw * cin   # im2col + GEMMs
    M = B * oh * ow
    gemm(layer.name, "fwd", M, cout, kcol, 0, 0, 0, bias=layer.bias)
    gemm(layer.name, "wgrad", cout, kcol, M // workers, 1, 1, 1, workers, _splits_tn(cout, kcol, M // workers, workers, deterministic))
    if not first:
      gemm(layer.name, "dgrad", M, kcol, cout, 0, 1, 0)
  return list(table.values())


def describe(p):
  if p["kind"] == "gemm":
    return "gemm %-5s M=%d N=%d K=%d%s%s" % (p["mode"], p["M"], p["N"], p["K"], " groups=%d" % p["groups"] if p["groups"] > 1 else "",
                                              " splits=%d" % p["splits"] if p["splits"] > 1 else "")
  return "conv%dx%d/s%d %-5s %dx%dx%d %d->%d%s%s" % (p["k"], p["k"], p["stride"], p["mode"], p["n"], p["h"], p["w"], p["cin"], p["cout"],
                                                    " groups=%d" % p["groups"] if p["groups"] > 1 else "", " splits=%d" % p["splits"] if p["splits"] > 1 else "")


# ---------------------------------------------------------------------------- #
# Activation traffic of the batch-norm and residual passes

FUSED_MB = (72, 40)   # single-launch batch norm envelope, forward / backward (`nn_native.set_bn_fused_limits` defaults; no ResNet-50 tensor is under its row minimum at these sizes)


def norm_layers(image_size):
  """[((C, H, W), relu, closes)] of every batch norm of ResNet-50 in forward order (closes: the closing norm of a residual unit,
  fused with the shortcut add and ReLU), and [(numel, shortcut kind)] of every residual unit."""
  from aggregathor_b200.engine.flat import FlatLayout
  from aggregathor_b200.models import Context, get_network
  from aggregathor_b200.models import core
  model = get_network("resnet_v1_50", 1000)
  layout, states = FlatLayout(), {}
  model.declare(layout, states)
  layout.freeze()
  params = torch.zeros(layout.padded_size)
  state = {k: torch.zeros(v) for k, v in states.items()}
  model.initialize(layout.views(params), state, torch.Generator().manual_seed(0))
  ctx = Context("torch", True, torch.float32, "cpu")
  ctx.master = ctx.weights = layout.views(params)
  ctx.state = state
  norms, units = [], []
  bn_forward, bn_closing, unit_forward = core.BatchNorm.forward, core.BatchNorm.forward_add_relu, core.Residual.forward

  def norm(self, x, c):
    norms.append((tuple(x.shape[1:]), self.relu, False))
    return bn_forward(self, x, c)

  def closing(self, x, shortcut, c):
    norms.append((tuple(x.shape[1:]), True, True))
    return bn_closing(self, x, shortcut, c)

  def unit(self, x, c):
    shortcut = self.shortcut
    kind = ("subsample" if shortcut.stride > 1 else "identity") if isinstance(shortcut, core.Subsample) else "projection"
    units.append((x[0].numel(), kind))
    return unit_forward(self, x, c)

  core.BatchNorm.forward, core.BatchNorm.forward_add_relu, core.Residual.forward = norm, closing, unit
  try:
    x = torch.zeros((1, 3, image_size, image_size)).contiguous(memory_format=torch.channels_last)
    with torch.no_grad():
      model.root.forward(x, ctx)
  finally:
    core.BatchNorm.forward, core.BatchNorm.forward_add_relu, core.Residual.forward = bn_forward, bn_closing, unit_forward
  return norms, units


def bn_pass(S, relu, closes, backward):
  """(pass name, activation bytes before, after) of one batch norm moving S-byte tensors, in one direction. A pass counts every
  activation it reads or writes once; per-channel vectors, and the single-launch kernel's L2 re-reads of rows past its on-chip
  stash, are left out."""
  extra = S if closes else 0     # forward: the shortcut read; backward: the masked gradient written for the shortcut
  if not backward:
    if S <= FUSED_MB[0] << 20:   # reads x (+ shortcut) once, writes y
      return "bn forward, single launch", 2 * S + extra, 2 * S + extra
    return "bn forward, pair", 3 * S + extra, 3 * S + extra   # statistics read x, apply reads x (+ shortcut) and writes y
  reads = 3 if relu else 2       # dy, x (, y for the mask)
  if S <= FUSED_MB[1] << 20:
    return "bn backward, single launch", (reads + 1) * S + extra, (reads + 1) * S + extra
  if relu and not closes:        # both passes recompute the mask from x: y is no longer read
    return "bn backward, pair, ReLU", (2 * reads + 1) * S, (2 * reads - 1) * S
  if closes:                     # the statistics pass stores the masked gradient; the apply reads it and x instead of dy, x and y
    return "bn backward, pair, closing", (2 * reads + 1) * S + extra, 2 * reads * S + extra
  return "bn backward, pair, no ReLU", (2 * reads + 1) * S, (2 * reads + 1) * S


def traffic(workers, batch, image_size):
  """HBM bytes per step of the batch-norm passes (single launch or statistics + apply pair, as the envelope picks) and of the
  residual-gradient passes, before and after summing the shortcut gradient in the data-gradient epilogue, recomputing the ReLU
  mask of the pair's backward from x and masking the closing norm's gradient once in the pair's backward (`bn_pass`).
  Returns {category: [tensors, before, after]}."""
  norms, units = norm_layers(image_size)
  B = workers * batch
  sums = collections.OrderedDict()

  def add(category, before, after):
    entry = sums.setdefault(category, [0, 0, 0])
    entry[0] += 1
    entry[1] += before
    entry[2] += after

  for shape, relu, closes in norms:
    S = 2 * B * math.prod(shape)
    for backward in (False, True):
      add(*bn_pass(S, relu, closes, backward))
  for numel, kind in units:
    X = 2 * B * numel
    if kind == "subsample":   # scatter into a full-size tensor (read X/4, write X) + add (2 reads, 1 write) -> in-place add of a quarter
      add("residual grads, subsample units", X // 4 + X + 3 * X, 3 * (X // 4))
    else:                     # add (2 reads, 1 write) -> the addend read by the data-gradient epilogue
      add("residual grads, %s units" % kind, 3 * X, X)
  return sums


# ---------------------------------------------------------------------------- #
# Timing

def launcher(p, device):
  """Closure that launches product `p` once on random operands (bf16; split-K accumulates into an output it never re-zeroes)."""
  from aggregathor_b200.ops import nn_native as nat
  bf = torch.bfloat16
  gen = torch.Generator(device=device).manual_seed(0)
  rnd = lambda *shape: torch.randn(shape, generator=gen, device=device, dtype=torch.float32).to(bf)
  if p["kind"] == "gemm":
    M, N, K, g = p["M"], p["N"], p["K"], p["groups"]
    ld = lambda c: (c + 7) // 8 * 8
    a = (rnd(K * g, ld(M)) if p["a_mn"] else rnd(M, ld(K)))[:, :(M if p["a_mn"] else K)]
    b = (rnd(K * g, ld(N)) if p["b_mn"] else rnd(N, ld(K)))[:, :(N if p["b_mn"] else K)]
    if g > 1:
      stride = (M * N + 63) // 64 * 64
      out = torch.zeros(g * stride, dtype=torch.float32, device=device)[:M * N].view(M, N)
    else:
      stride = 0
      out = nat.alloc_out(M, N, torch.float32 if p["out_fp32"] else bf, device)
    bias = torch.randn(N, device=device) if p["bias"] else None
    return lambda: nat._gemm(a, b, out, M, N, K, p["a_mn"], p["b_mn"], bias, False, p["splits"], 0, g, stride), out
  n, h, w, oh, ow, cin, cout, k = (p[key] for key in ("n", "h", "w", "oh", "ow", "cin", "cout", "k"))
  mode, g = ("fwd", "dgrad", "wgrad").index(p["mode"]), p["groups"]
  x, y, wt = rnd(n, h, w, cin), rnd(n, oh, ow, cout), rnd(cout, k, k, cin)
  if mode == 0:
    act, other, out = x, wt, torch.empty_like(y)
  elif mode == 1:
    act, other, out = y, wt, torch.empty_like(x)
  else:
    stride = (cout * k * k * cin + 63) // 64 * 64
    act, other, out = y, x, torch.zeros(g * stride, dtype=torch.float32, device=device)
  gs = stride if mode == 2 else 0
  return lambda: nat._conv_implicit(mode, act, other, out, n, h, w, oh, ow, cin, cout, k, p["stride"], p["pads"], splits=p["splits"], groups=g, group_stride=gs), out


def time_window(fn, launches):
  begin, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  begin.record()
  for _ in range(launches):
    fn()
  end.record()
  end.synchronize()
  return begin.elapsed_time(end) / launches


def run_products(args):
  from aggregathor_b200.ops import nn_native as nat
  global SM_COUNT
  device = torch.device("cuda", 0)
  torch.cuda.set_device(device)
  SM_COUNT = torch.cuda.get_device_properties(device).multi_processor_count
  lib = nat._lib()
  table = products(args.workers, args.batch_size, args.image_size, nat._DETERMINISTIC)
  rows = []
  for p in table:
    fn, out = launcher(p, device)
    per = {}
    for staged in (0, 1):   # warm-up of both epilogues, and a launch count that fills a window
      lib.agb_gemm_set_epilogue(staged)
      for _ in range(3):
        fn()
      per[staged] = time_window(fn, 3)
    launches = max(10, int(args.seconds * 1e3 / max(min(per.values()), 1e-3)))
    samples = {0: [], 1: []}
    for _ in range(2):
      for staged in (0, 1):
        lib.agb_gemm_set_epilogue(staged)
        samples[staged].append(time_window(fn, launches))
    if p["splits"] == 1:   # same output under both epilogues (split-K sums arrive in varying order)
      lib.agb_gemm_set_epilogue(0)
      fn()
      ref = out.clone()
      lib.agb_gemm_set_epilogue(1)
      fn()
      torch.cuda.synchronize()
      p["bit_identical"] = bool(torch.equal(ref, out))
    regs, staged = min(samples[0]), min(samples[1])
    row = dict(p, product=describe(p), regs_ms=regs, staged_ms=staged, regs_samples=samples[0], staged_samples=samples[1], launches=launches,
               tflops_staged=p["flop"] / staged / 1e9, tbs_staged=p["bytes"] / staged / 1e9, tflops_regs=p["flop"] / regs / 1e9, tbs_regs=p["bytes"] / regs / 1e9)
    rows.append(row)
    print("%-58s x%-3d regs %8.4f ms  staged %8.4f ms  (%+.1f %%)  %6.1f TFLOP/s %5.2f TB/s%s" % (
      row["product"], p["calls"], regs, staged, 100 * (staged / regs - 1), row["tflops_staged"], row["tbs_staged"],
      "" if p.get("bit_identical", True) else "  OUTPUTS DIFFER"), flush=True)
    del fn, out
    torch.cuda.empty_cache()
  lib.agb_gemm_set_epilogue(1)
  total_regs = sum(r["regs_ms"] * r["calls"] for r in rows)
  total_staged = sum(r["staged_ms"] * r["calls"] for r in rows)
  return {"card": card(), "products": rows, "step_ms_regs": total_regs, "step_ms_staged": total_staged}


# ---------------------------------------------------------------------------- #
# Step profile

def run_profile(args):
  """Kernel time of the headline step grouped by kernel name (torch.profiler, CUDA activities)."""
  from torch.profiler import ProfilerActivity, profile
  from aggregathor_b200 import aggregators, experiments
  from aggregathor_b200.engine.trainer import Manager
  device = torch.device("cuda", 0)
  torch.cuda.set_device(device)
  exp = experiments.instantiate("slim-resnet_v1_50-imagenet", ["batch-size:%d" % args.batch_size, "synthetic-samples:%d" % max(256, 4 * args.batch_size)])
  gar = aggregators.instantiate("krum", args.workers, 2, [])
  manager = Manager(exp, gar, args.workers, "sgd", [], "fixed", ["initial-rate:0.01"], device=device, engine="fused", backend="auto", seed=0)
  for _ in range(3):
    manager.train()
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    begin = time.perf_counter()
    for _ in range(args.steps):
      manager.train()
    torch.cuda.synchronize()
    wall = time.perf_counter() - begin
  manager.close()
  by_name = collections.defaultdict(lambda: [0.0, 0])
  for event in prof.events():
    if event.device_type == torch.autograd.DeviceType.CUDA:
      by_name[event.name][0] += event.device_time_total / 1e3 / args.steps
      by_name[event.name][1] += 1
  kernels = sorted(({"name": k, "ms_per_step": v[0], "calls_per_step": v[1] / args.steps} for k, v in by_name.items()), key=lambda r: -r["ms_per_step"])
  total = sum(r["ms_per_step"] for r in kernels)
  family = lambda r: "gemm_sm90_kernel" in r["name"] or "conv_sm90_kernel" in r["name"]
  gemm_ms = sum(r["ms_per_step"] for r in kernels if family(r))
  os.makedirs(args.out, exist_ok=True)
  prof.export_chrome_trace(os.path.join(args.out, "step_trace.json"))
  result = {"card": card(), "epilogue": os.environ.get("AGB_GEMM_EPILOGUE", "staged"), "wall_ms_per_step_profiled": wall * 1e3 / args.steps,
            "kernel_ms_per_step": total, "gemm_family_ms_per_step": gemm_ms, "gemm_family_share": gemm_ms / total if total else None, "kernels": kernels}
  print("kernel time %.2f ms/step, GEMM family %.2f ms (%.1f %%), profiled wall %.2f ms/step" % (total, gemm_ms, 100 * gemm_ms / max(total, 1e-9), wall * 1e3 / args.steps))
  for r in kernels[:25]:
    print("  %8.3f ms  %6.1f calls  %s" % (r["ms_per_step"], r["calls_per_step"], r["name"][:150]))
  return result


def main():
  args = parse()
  if args.traffic:
    sums = traffic(args.workers, args.batch_size, args.image_size)
    print("%-42s %7s %10s %10s %9s" % ("pass (%d images, bf16)" % (args.workers * args.batch_size), "tensors", "before GB", "after GB", "saved GB"))
    for category, (count, before, after) in sums.items():
      print("%-42s %7d %10.2f %10.2f %9.2f" % (category, count, before / 1e9, after / 1e9, (before - after) / 1e9))
    before, after = sum(v[1] for v in sums.values()), sum(v[2] for v in sums.values())
    print("%-42s %7s %10.2f %10.2f %9.2f" % ("total", "", before / 1e9, after / 1e9, (before - after) / 1e9))
    return 0
  if args.dry_run:
    table = products(args.workers, args.batch_size, args.image_size)
    flop = sum(p["flop"] * p["calls"] for p in table)
    print("%d distinct products, %d calls, %.2f TFLOP and %.1f GB per step (operands once, outputs once)" % (
      len(table), sum(p["calls"] for p in table), flop / 1e12, sum(p["bytes"] * p["calls"] for p in table) / 1e9))
    for p in table:
      print("%-58s x%-3d %9.1f GFLOP %8.1f MB  %5.0f FLOP/B" % (describe(p), p["calls"], p["flop"] / 1e9, p["bytes"] / 1e6, p["flop"] / p["bytes"]))
    return 0
  if not torch.cuda.is_available():
    raise SystemExit("nn_bench.py needs a CUDA device (use --dry-run for the product table)")
  os.makedirs(args.out, exist_ok=True)
  result = run_profile(args) if args.profile else run_products(args)
  name = "profile_%s.json" % result["epilogue"] if args.profile else "products.json"
  with open(os.path.join(args.out, name), "w") as f:
    json.dump(result, f, indent=1, default=str)
  if not args.profile:
    print("sum over the step: regs %.2f ms, staged %.2f ms; card %s" % (result["step_ms_regs"], result["step_ms_staged"], json.dumps(result["card"])))
  return 0


if __name__ == "__main__":
  sys.exit(main())

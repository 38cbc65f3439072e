#!/usr/bin/env python3
"""Batch-norm passes of the headline step (slim ResNet-50 v1, n = 8 batched logical workers x 32 images, 224x224, bf16): every
distinct pass at its batched shape, its activation bytes (the accounting of `nn_bench.py --traffic`), its device time and the
bandwidth it reaches.

    python benchmarks/bn_bench.py --dry-run          # shape and byte table (no GPU needed)
    python benchmarks/bn_bench.py --out DIR          # time every pass; results go to DIR/bn_passes.json

A pass is one batch-norm call as the training step makes it, with one group per logical worker: the statistics + apply pair
(forward; backward with the ReLU mask recomputed from x; backward without ReLU; backward of the closing norm of a residual unit,
which also returns the masked gradient for the shortcut) or the single-launch kernel. Its time is taken with CUDA events over a
window of at least `--seconds` after warm-up; the split between its kernels comes from a separate torch.profiler window of the
same length. TB/s is bytes over time, and its share is against the 3.35 TB/s HBM3 bandwidth of NVIDIA's H100 SXM data sheet.
"""

import argparse
import collections
import json
import math
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import torch  # noqa: E402

import nn_bench  # noqa: E402

PEAK_TBS = 3.35   # H100 SXM HBM3, data sheet


def parse():
  parser = argparse.ArgumentParser()
  parser.add_argument("--dry-run", action="store_true")
  parser.add_argument("--out", type=str, default="bn_bench_out")
  parser.add_argument("--workers", type=int, default=8)
  parser.add_argument("--batch-size", type=int, default=32, help="per logical worker")
  parser.add_argument("--image-size", type=int, default=224)
  parser.add_argument("--seconds", type=float, default=0.25, help="length of one timing window")
  return parser.parse_args()


def passes(workers, batch, image_size):
  """Distinct passes of one step: [dict(category, shape (C, H, W), relu, closes, backward, bytes, calls)] in first-use order."""
  B = workers * batch
  norms, _ = nn_bench.norm_layers(image_size)
  table = collections.OrderedDict()
  for shape, relu, closes in norms:
    S = 2 * B * math.prod(shape)
    for backward in (False, True):
      category, _, after = nn_bench.bn_pass(S, relu, closes, backward)
      key = (category, shape, relu, closes, backward)
      if key not in table:
        table[key] = dict(category=category, shape=shape, relu=relu, closes=closes, backward=backward, bytes=after, calls=0)
      table[key]["calls"] += 1
  return list(table.values())


def describe(p):
  c, h, w = p["shape"]
  return "%-28s %4dx%-3d C=%-4d%s%s" % (p["category"], h, w, c, " relu" if p["relu"] and not p["closes"] else "", " +shortcut" if p["closes"] else "")


def launcher(p, workers, batch, device):
  """Closure that runs pass `p` once on random bf16 operands, as the training step calls it."""
  from aggregathor_b200.ops import nn_native as nat
  gen = torch.Generator(device=device).manual_seed(0)
  c, h, w = p["shape"]
  groups = workers
  shape = (workers * batch, c, h, w)
  rnd = lambda: torch.randn(shape, generator=gen, device=device).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
  gamma, beta = 1 + 0.1 * torch.randn(c, generator=gen, device=device), 0.1 * torch.randn(c, generator=gen, device=device)
  mm, mv = torch.zeros(c, device=device), torch.ones(c, device=device)
  x = rnd()
  shortcut = rnd() if p["closes"] else None
  relu = p["relu"]
  if not p["backward"]:
    if p["closes"]:
      return lambda: nat.batchnorm_forward(x, gamma, beta, mm, mv, 0.9, 1e-5, True, groups, shortcut)
    return lambda: nat.batchnorm_forward(x, gamma, beta, mm, mv, 0.9, 1e-5, relu, groups, coef=True)
  if p["closes"]:
    y, mean, rstd = nat.batchnorm_forward(x, gamma, beta, mm, mv, 0.9, 1e-5, True, groups, shortcut)
    coef = None
  else:
    y, mean, rstd, coef = nat.batchnorm_forward(x, gamma, beta, mm, mv, 0.9, 1e-5, relu, groups, coef=True)
  dy = rnd()
  grads = torch.zeros((2, groups, c), device=device)
  if p["closes"]:
    return lambda: nat.batchnorm_backward(dy, x, y, gamma, mean, rstd, True, grads[0, 0], grads[1, 0], groups, c, want_masked=True)
  return lambda: nat.batchnorm_backward(dy, x, y, gamma, mean, rstd, relu, grads[0, 0], grads[1, 0], groups, c, mask_coef=coef if relu else None)


def kernel_split(fn, launches):
  """{kernel name: ms per pass} over `launches` passes (torch.profiler, CUDA activities)."""
  from torch.profiler import ProfilerActivity, profile
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(launches):
      fn()
    torch.cuda.synchronize()
  split = collections.defaultdict(float)
  for event in prof.events():
    if event.device_type == torch.autograd.DeviceType.CUDA:
      split[event.name] += event.device_time_total / 1e3 / launches
  return dict(split)


def short(name):
  """Kernel name with its template arguments, without its return type and argument list."""
  name = name.replace("(anonymous namespace)::", "")
  name = name[5:] if name.startswith("void ") else name
  return name.split("(")[0]


def run(args):
  from aggregathor_b200.ops import nn_native as nat  # noqa: F401  (builds / loads the native library before any timing)
  device = torch.device("cuda", 0)
  torch.cuda.set_device(device)
  card_before = nn_bench.card()
  rows = []
  for p in passes(args.workers, args.batch_size, args.image_size):
    fn = launcher(p, args.workers, args.batch_size, device)
    for _ in range(3):
      fn()
    estimate = nn_bench.time_window(fn, 3)
    launches = max(10, int(math.ceil(args.seconds * 1e3 / max(estimate, 1e-3))))
    samples = [nn_bench.time_window(fn, launches) for _ in range(2)]
    ms = min(samples)
    split = kernel_split(fn, launches)
    row = dict(p, shape=list(p["shape"]), pass_name=describe(p), ms=ms, samples=samples, launches=launches, window_s=ms * launches / 1e3,
               tbs=p["bytes"] / ms / 1e9, kernels={short(k): v for k, v in split.items()})
    row["peak_share"] = row["tbs"] / PEAK_TBS
    rows.append(row)
    print("%-58s x%-2d %8.1f MB %8.4f ms %5.2f TB/s (%4.1f %%)  %s" % (
      row["pass_name"], p["calls"], p["bytes"] / 1e6, ms, row["tbs"], 100 * row["peak_share"],
      "  ".join("%s %.4f" % (k, v) for k, v in sorted(row["kernels"].items(), key=lambda kv: -kv[1]))), flush=True)
    del fn
    torch.cuda.empty_cache()
  summary = collections.OrderedDict()
  for r in rows:
    s = summary.setdefault(r["category"], dict(tensors=0, bytes=0, ms=0.0, kernels=collections.defaultdict(float)))
    s["tensors"] += r["calls"]
    s["bytes"] += r["bytes"] * r["calls"]
    s["ms"] += r["ms"] * r["calls"]
    for k, v in r["kernels"].items():
      s["kernels"][k] += v * r["calls"]
  print("\nper step %-33s %7s %9s %9s %7s %6s" % ("", "tensors", "GB", "ms", "TB/s", "peak"))
  for category, s in summary.items():
    s["tbs"] = s["bytes"] / s["ms"] / 1e9
    s["peak_share"] = s["tbs"] / PEAK_TBS
    print("  %-40s %7d %9.2f %9.3f %7.2f %5.1f %%" % (category, s["tensors"], s["bytes"] / 1e9, s["ms"], s["tbs"], 100 * s["peak_share"]))
    for k, v in sorted(s["kernels"].items(), key=lambda kv: -kv[1]):
      print("      %9.3f ms  %s" % (v, k))
  card_after = nn_bench.card()
  print("card: %s (after: %s)" % (json.dumps(card_before), json.dumps(card_after)))
  return {"card": card_before, "card_after": card_after, "peak_tbs": PEAK_TBS, "passes": rows, "per_step": summary}


def main():
  args = parse()
  if args.dry_run:
    table = passes(args.workers, args.batch_size, args.image_size)
    print("%-58s %5s %10s %10s" % ("pass (%d images, bf16, %d groups)" % (args.workers * args.batch_size, args.workers), "calls", "MB / call", "GB / step"))
    for p in table:
      print("%-58s %5d %10.1f %10.2f" % (describe(p), p["calls"], p["bytes"] / 1e6, p["bytes"] * p["calls"] / 1e9))
    print("total %.2f GB per step over %d distinct passes" % (sum(p["bytes"] * p["calls"] for p in table) / 1e9, len(table)))
    return 0
  if not torch.cuda.is_available():
    raise SystemExit("bn_bench.py needs a CUDA device (use --dry-run for the shape and byte table)")
  result = run(args)
  os.makedirs(args.out, exist_ok=True)
  with open(os.path.join(args.out, "bn_passes.json"), "w") as f:
    json.dump(result, f, indent=1, default=str)
  return 0


if __name__ == "__main__":
  sys.exit(main())

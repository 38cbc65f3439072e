#!/usr/bin/env python3
"""Cost of divide-and-conquer (`dnc`) on one GPU, next to Krum.

1. The fused step of `krum` and `dnc` (SGD, d = ResNet-50's by default, n = 8, f = 2), with and without NNM: the engines of all the
   configurations are built first, then timed round by round in turn (5 rounds of `--iters` steps), so clock and thermal drift hit
   every configuration alike; medians in ms per step.
2. The DnC selection alone at n = 32, on the stand-alone op over a small d (`--small-dim`), where the step is dominated by fixed
   costs: `average` (launch, one pass), `dnc` with 1 sampled coordinate (adds the gather, the exchange and the float64 Jacobi on
   32 rows) and `dnc` with `--subsample` coordinates (adds the sampled distance pass). The differences estimate the Jacobi and the
   sampled pass; medians over 5 rounds of `--iters` calls.
Prints one JSON object, and writes it to `--out` when given.
"""

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from aggregathor_b200 import aggregators  # noqa: E402
from aggregathor_b200.aggregators import FusedSpec  # noqa: E402
from aggregathor_b200.engine.flat import FlatLayout  # noqa: E402
from aggregathor_b200.engine.optimizers import optimizers  # noqa: E402
from aggregathor_b200.engine.schedules import build  # noqa: E402
from aggregathor_b200.ops import gar as gar_ops  # noqa: E402
from aggregathor_b200.parallel.aggregation import FusedAggregation  # noqa: E402


def timed(fn, iters):
  torch.cuda.synchronize()
  begin, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  begin.record()
  for _ in range(iters):
    fn()
  end.record()
  torch.cuda.synchronize()
  return begin.elapsed_time(end) / iters


def alternated(fns, iters, rounds=5):
  for fn in fns.values():
    for _ in range(3):
      fn()
  samples = {name: [] for name in fns}
  for _ in range(rounds):
    for name, fn in fns.items():
      samples[name].append(timed(fn, iters))
  return {name: sorted(values)[len(values) // 2] for name, values in samples.items()}, samples


def main():
  parser = argparse.ArgumentParser()
  parser.add_argument("--dim", type=int, default=25557032)
  parser.add_argument("--small-dim", type=int, default=40000)
  parser.add_argument("--subsample", type=int, default=10000)
  parser.add_argument("--iters", type=int, default=10)
  parser.add_argument("--out", type=str, default=None)
  args = parser.parse_args()
  device = torch.device("cuda", 0)
  torch.cuda.set_device(device)
  n, f = 8, 2
  layout = FlatLayout()
  layout.add("theta", (args.dim,))
  layout.freeze()
  d = layout.padded_size
  grads = torch.randn((n, d), device=device, generator=torch.Generator(device=device).manual_seed(3))
  grads[n - f:].mul_(20.0).add_(3.0)
  engines = {}
  for rule, extra in (("krum", []), ("dnc", ["subsample:%d" % args.subsample])):
    for mix in ("none", "nnm"):
      gar = aggregators.instantiate(rule, n, f, extra)
      engine = FusedAggregation(gar, layout, n, build(optimizers, "optimizer", "sgd", []), device=device, pre_aggregation=mix, nb_decl_byz=f)
      engine.grads.copy_(grads)
      engines["%s%s" % (rule, "" if mix == "none" else "+nnm")] = engine
  step_ms, step_rounds = alternated({name: (lambda e=engine: e.step(0.01)) for name, engine in engines.items()}, args.iters)
  del engines
  torch.cuda.empty_cache()
  m = 32
  G = torch.randn((m, args.small_dim), device=device, generator=torch.Generator(device=device).manual_seed(4))
  specs = {"average": FusedSpec("average", m), "dnc_b1": FusedSpec("dnc", m, f=8, iterations=1, subsample=1),
           "dnc_b": FusedSpec("dnc", m, f=8, iterations=1, subsample=args.subsample)}
  small_ms, small_rounds = alternated({name: (lambda s=spec: gar_ops.aggregate(s, G, step=1)) for name, spec in specs.items()}, args.iters)
  props = torch.cuda.get_device_properties(device)
  report = {"gpu": props.name, "n": n, "f": f, "d": d, "subsample": args.subsample, "fused_step_ms": step_ms, "fused_step_rounds_ms": step_rounds,
            "n32": {"d": args.small_dim, "median_ms": small_ms, "rounds_ms": small_rounds,
                    "jacobi_and_exchange_ms": small_ms["dnc_b1"] - small_ms["average"], "sampled_pass_ms": small_ms["dnc_b"] - small_ms["dnc_b1"]}}
  print(json.dumps(report))
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fd:
      json.dump(report, fd, indent=1)


if __name__ == "__main__":
  main()

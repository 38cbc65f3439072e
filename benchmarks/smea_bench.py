#!/usr/bin/env python3
"""Cost of smallest maximum eigenvalue averaging (`smea`) on one GPU, next to Krum and MDA.

1. The fused step of `smea`, `krum` and `mda` (SGD, d = ResNet-50's by default, n = 8, f = 2), with and without NNM: the engines of all
   the configurations are built first, then timed round by round in turn (5 rounds of `--iters` steps), so clock and thermal drift hit
   every configuration alike; medians in ms per step.
2. The SMEA selection alone on the stand-alone op over a small d (`--small-dim`), for (n, f) in (8, 2), (16, 4), (26, 4), (32, 3)
   (the largest sets of 22 and 29 rows the bound C(n, f) <= 2^14 admits): `krum`
   runs the same distance pass, exchange and mean, so `smea` - `krum` estimates the search over the C(n, f) sets (one float64 Jacobi
   each); medians over 5 rounds of `--iters` calls.
The card's name, power limit and SM clock are read in the same run. Prints one JSON object, and writes it to `--out` when given.
"""

import argparse
import json
import math
import os
import subprocess
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


def card():
  """Name, power limit and SM clocks of GPU 0, as nvidia-smi reports them (read-only query)."""
  fields = "name,power.limit,clocks.sm,clocks.max.sm"
  try:
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + fields, "--format=csv,noheader"], stdout=subprocess.PIPE,
                         stderr=subprocess.STDOUT, timeout=60).stdout.decode().strip()
  except (OSError, subprocess.SubprocessError) as err:
    out = "unavailable: %s" % err
  return {"query": fields, "value": out}


def main():
  parser = argparse.ArgumentParser()
  parser.add_argument("--dim", type=int, default=25557032)
  parser.add_argument("--small-dim", type=int, default=40000)
  parser.add_argument("--iters", type=int, default=10)
  parser.add_argument("--out", type=str, default=None)
  args = parser.parse_args()
  device = torch.device("cuda", 0)
  torch.cuda.set_device(device)
  before = card()
  n, f = 8, 2
  layout = FlatLayout()
  layout.add("theta", (args.dim,))
  layout.freeze()
  d = layout.padded_size
  grads = torch.randn((n, d), device=device, generator=torch.Generator(device=device).manual_seed(3))
  grads[n - f:].mul_(20.0).add_(3.0)
  engines = {}
  for rule in ("krum", "mda", "smea"):
    for mix in ("none", "nnm"):
      gar = aggregators.instantiate(rule, n, f, [])
      engine = FusedAggregation(gar, layout, n, build(optimizers, "optimizer", "sgd", []), device=device, pre_aggregation=mix, nb_decl_byz=f)
      engine.grads.copy_(grads)
      engines["%s%s" % (rule, "" if mix == "none" else "+nnm")] = engine
  step_ms, step_rounds = alternated({name: (lambda e=engine: e.step(0.01)) for name, engine in engines.items()}, args.iters)
  del engines
  torch.cuda.empty_cache()
  selection = {}
  for sn, sf in ((8, 2), (16, 4), (26, 4), (32, 3)):
    G = torch.randn((sn, args.small_dim), device=device, generator=torch.Generator(device=device).manual_seed(sn + sf))
    specs = {"krum": FusedSpec("krum", sn, f=sf, m=sn - sf), "smea": FusedSpec("smea", sn, f=sf)}
    ms, rounds = alternated({name: (lambda s=spec: gar_ops.aggregate(s, G)) for name, spec in specs.items()}, args.iters)
    selection["%d,%d" % (sn, sf)] = {"sets": math.comb(sn, sf), "median_ms": ms, "rounds_ms": rounds, "selection_ms": ms["smea"] - ms["krum"]}
  report = {"gpu": torch.cuda.get_device_properties(device).name, "card_before": before, "card_after": card(), "n": n, "f": f, "d": d,
            "fused_step_ms": step_ms, "fused_step_rounds_ms": step_rounds, "small_dim": args.small_dim, "selection": selection}
  print(json.dumps(report))
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fd:
      json.dump(report, fd, indent=1)


if __name__ == "__main__":
  main()

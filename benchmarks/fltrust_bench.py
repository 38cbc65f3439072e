#!/usr/bin/env python3
"""Cost of FLTrust (`fltrust`) on one GPU: the full training step of the flagship workload (ResNet-50, 8 workers of batch 32, f = 2,
SGD, fused engine) under `krum` and under `fltrust`.

FLTrust adds, per step, one unbatched forward/backward of rank 0 on a batch of the root dataset, and its aggregation reads n + 1 rows
(sums pass) then n rows (weighted sum) where Krum reads n rows twice. Both managers are built first and warmed up (graph capture
included), then timed round by round in turn (`--rounds` rounds of `--steps` steps each, CUDA events around the steps), so clock and
thermal drift hit both alike; medians in ms per step. The card's name, power limit and SM clocks are read in the same run. Prints one
JSON object, and writes it to `--out` when given.
"""

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from aggregathor_b200 import aggregators, experiments  # noqa: E402
from aggregathor_b200.engine.trainer import Manager  # noqa: E402


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
  parser = argparse.ArgumentParser(description=__doc__.splitlines()[0])
  parser.add_argument("--model", default="resnet_v1_50")
  parser.add_argument("--batch-size", type=int, default=32)
  parser.add_argument("--nb-workers", type=int, default=8)
  parser.add_argument("--nb-decl-byz-workers", type=int, default=2)
  parser.add_argument("--root-size", type=int, default=100)
  parser.add_argument("--steps", type=int, default=20)
  parser.add_argument("--warmup", type=int, default=4)
  parser.add_argument("--rounds", type=int, default=5)
  parser.add_argument("--out", default="")
  args = parser.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("fltrust_bench.py measures on a GPU: none is visible")
  device = torch.device("cuda", 0)
  torch.cuda.set_device(device)
  n, f = args.nb_workers, args.nb_decl_byz_workers
  exp_args = ["batch-size:%d" % args.batch_size, "synthetic-samples:%d" % max(256, 4 * args.batch_size, args.root_size)]
  managers = {}
  for rule, rule_args in (("krum", []), ("fltrust", ["root-size:%d" % args.root_size])):
    experiment = experiments.instantiate("slim-%s-imagenet" % args.model, exp_args)
    managers[rule] = Manager(experiment, aggregators.instantiate(rule, n, f, rule_args), n, "sgd", [], "fixed", ["initial-rate:0.01"],
                             device=device, engine="fused", seed=0)
  for manager in managers.values():
    for _ in range(args.warmup):
      manager.train()
  torch.cuda.synchronize()

  def timed(manager):
    torch.cuda.synchronize()
    begin, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    begin.record()
    for _ in range(args.steps):
      manager.train()
    end.record()
    torch.cuda.synchronize()
    return begin.elapsed_time(end) / args.steps

  rounds = {rule: [] for rule in managers}
  for _ in range(args.rounds):
    for rule, manager in managers.items():
      rounds[rule].append(timed(manager))
  median = lambda values: sorted(values)[len(values) // 2]
  result = {"benchmark": "fltrust", "model": args.model, "n": n, "f": f, "batch_size": args.batch_size, "root_size": args.root_size,
            "d": managers["krum"].layout.size, "engine": managers["fltrust"].aggregation.name,
            "whole_step_graph": {rule: bool(m._graph_whole) for rule, m in managers.items()},
            "ms_per_step": {rule: median(v) for rule, v in rounds.items()}, "rounds_ms": rounds,
            "final_loss": {rule: float(m.total_loss) for rule, m in managers.items()}, "card": card()}
  result["fltrust_overhead_ms"] = result["ms_per_step"]["fltrust"] - result["ms_per_step"]["krum"]
  for manager in managers.values():
    manager.close()
  text = json.dumps(result)
  print(text)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fd:
      fd.write(text + "\n")


if __name__ == "__main__":
  main()

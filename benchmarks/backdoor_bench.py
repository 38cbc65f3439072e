#!/usr/bin/env python3
"""Cost of the backdoor attack (`--attack backdoor`) on one GPU: the full training step (fused engine, Krum with f = 2, SGD) with no attack,
with `label-flip` and with `backdoor` (scale:4), each with k = 2 real Byzantine workers.

The backdoor adds no launch and no pass: the trigger is one predicate per pixel in the input kernel (`image_normalize` for the synthetic
ImageNet of ResNet-50, the preprocessing kernel for cnnet) and the relabelling and scaling are a few parameters of the softmax
cross-entropy kernel. Two configurations: ResNet-50 on synthetic ImageNet and cnnet on CIFAR-10 with its preprocessing kernel, 8
workers of batch 32 each. All managers of a configuration are built first and warmed up (graph capture included), then timed round by
round in turn (`--rounds` rounds of `--steps` steps each, CUDA events around the steps), so clock and thermal drift hit them alike; medians
in ms per step, and the native kernel launches per step. The card's name, power limit and SM clocks are read in the same run. Prints one
JSON object, and writes it to `--out` when given.
"""

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from aggregathor_b200 import aggregators, attacks, experiments  # noqa: E402
from aggregathor_b200.engine.trainer import Manager  # noqa: E402
from aggregathor_b200.ops import counters  # noqa: E402

ATTACKS = {"none": None, "label-flip": [], "backdoor": ["target:0", "scale:4"]}
CONFIGS = {"resnet50": ("slim-resnet_v1_50-imagenet", ["synthetic-samples:256"]), "cnnet": ("cnnet", [])}


def card():
  """Name, power limit and SM clocks of GPU 0, as nvidia-smi reports them (read-only query)."""
  fields = "name,power.limit,clocks.sm,clocks.max.sm"
  try:
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + fields, "--format=csv,noheader"], stdout=subprocess.PIPE,
                         stderr=subprocess.STDOUT, timeout=60).stdout.decode().strip()
  except (OSError, subprocess.SubprocessError) as err:
    out = "unavailable: %s" % err
  return {"query": fields, "value": out}


def measure(config, args, device):
  experiment, exp_args = CONFIGS[config]
  n, k = args.nb_workers, 2
  managers = {}
  for name, attack_args in ATTACKS.items():
    attack = attacks.instantiate(name, n, k, attack_args) if attack_args is not None else None
    managers[name] = Manager(experiments.instantiate(experiment, ["batch-size:%d" % args.batch_size] + exp_args), aggregators.instantiate("krum", n, 2, []), n,
                             "sgd", [], "fixed", ["initial-rate:0.01"], device=device, engine="fused", seed=0, attack=attack,
                             nb_real_byz=k if attack is not None else 0)
  for manager in managers.values():
    for _ in range(args.warmup):
      manager.train()
  torch.cuda.synchronize()

  def timed(manager):
    torch.cuda.synchronize()
    begin, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    launches = counters.launches
    begin.record()
    for _ in range(args.steps):
      manager.train()
    end.record()
    torch.cuda.synchronize()
    return begin.elapsed_time(end) / args.steps, (counters.launches - launches) // args.steps

  rounds, launches = {name: [] for name in managers}, {}
  for _ in range(args.rounds):
    for name, manager in managers.items():
      ms, launches[name] = timed(manager)
      rounds[name].append(ms)
  median = lambda values: sorted(values)[len(values) // 2]
  result = {"experiment": experiment, "d": managers["none"].layout.size, "engine": managers["none"].aggregation.name,
            "whole_step_graph": {name: bool(m._graph_whole) for name, m in managers.items()},
            "ms_per_step": {name: median(v) for name, v in rounds.items()}, "rounds_ms": rounds, "gpu_launches": launches,
            "spread_ms": {name: max(v) - min(v) for name, v in rounds.items()},
            "final_loss": {name: float(m.total_loss) for name, m in managers.items()}}
  for manager in managers.values():
    manager.close()
  return result


def main():
  parser = argparse.ArgumentParser(description=__doc__.splitlines()[0])
  parser.add_argument("--configs", default=",".join(CONFIGS))
  parser.add_argument("--batch-size", type=int, default=32)
  parser.add_argument("--nb-workers", type=int, default=8)
  parser.add_argument("--steps", type=int, default=20)
  parser.add_argument("--warmup", type=int, default=4)
  parser.add_argument("--rounds", type=int, default=5)
  parser.add_argument("--out", default="")
  args = parser.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("backdoor_bench.py measures on a GPU: none is visible")
  device = torch.device("cuda", 0)
  torch.cuda.set_device(device)
  result = {"benchmark": "backdoor", "n": args.nb_workers, "k": 2, "f": 2, "batch_size": args.batch_size, "steps": args.steps, "rounds": args.rounds,
            "card": card()}
  for config in args.configs.split(","):
    result[config] = measure(config, args, device)
    torch.cuda.empty_cache()
  result["card_after"] = card()
  text = json.dumps(result)
  print(text)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fd:
      fd.write(text + "\n")


if __name__ == "__main__":
  main()

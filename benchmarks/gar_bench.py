#!/usr/bin/env python3
"""Aggregation-path micro-benchmark + cross-engine check (1..8 GPUs, launch with torchrun for N > 1).

For every rule: run the fused engine and the baseline engine (NCCL all-gather + stand-alone kernel + SGD kernel) from
identical parameters/gradients, check that (a) both produce the same parameters (tolerance) and (b) every rank ends
with bit-identical parameters (checksum), then time each engine's step with CUDA events (max over ranks).
Reports, per rule: ms per step for both engines, the bytes that must cross NVLink into each GPU, GB/s and the
fraction of the peer-copy rate measured at start-up; writes JSON to <--gar-out>/gar_bench_<N>.json.

`--gar-attack alie|ipm`: the last f workers are omniscient Byzantine workers. Every step of both engines first crafts their rows
(`craft_byzantine`: the sm_90a kernel, sharded over the ranks on the fused engine, after the NCCL all-gather on the baseline one);
the crafting kernel is also timed alone, next to the torch reference on the same device, with the (H + k) * d * 4 bytes it must move.
`--gar-dump-rows` then saves, from the last rank, every row the fused engine aggregated (honest and crafted, all d coordinates).
`--gar-rule-args key:value ...` passes the same `--aggregator-args` to every rule (rules ignore keys they do not use). The
`geometric-median` and `centered-clipping` entries also report their T + 1 passes' (T + 1) * n * slice * 4 bytes and their rate.
`--gar-worker-momentum beta` also times the worker-momentum kernel alone on the [w, d] rows of a rank (`ops.gar.worker_momentum_`,
dampening 0), with the 16 * w * d bytes it must move (G and M read and written once).
"""

import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from aggregathor_b200 import aggregators, attacks, tools  # noqa: E402
from aggregathor_b200.aggregators import _ops  # noqa: E402
from aggregathor_b200.engine.flat import FlatLayout  # noqa: E402
from aggregathor_b200.engine.optimizers import optimizers  # noqa: E402
from aggregathor_b200.engine.schedules import build  # noqa: E402
from aggregathor_b200.ops import gar as gar_ops  # noqa: E402
from aggregathor_b200.parallel.aggregation import BaselineAggregation, FusedAggregation  # noqa: E402


def main():
  parser = argparse.ArgumentParser()
  parser.add_argument("--gar-dim", dest="d", type=int, default=25557032)
  parser.add_argument("--gar-workers", dest="nb_workers", type=int, default=8)
  parser.add_argument("--gar-iters", dest="iters", type=int, default=10)
  parser.add_argument("--gar-rules", dest="rules", type=str, default="average,average-nan,median,averaged-median,krum,bulyan")
  parser.add_argument("--gar-out", dest="out", type=str, default=".")
  parser.add_argument("--gar-byz", dest="byz", type=int, default=None, help="declared Byzantine workers f of every rule (default: 1 for Bulyan below 11 workers, else 2)")
  parser.add_argument("--gar-attack", dest="attack", choices=("alie", "ipm"), default=None, help="omniscient attack by the last f workers, crafted every step")
  parser.add_argument("--gar-dump-rows", dest="dump_rows", action="store_true", help="with --gar-attack: save the last rank's view of every row to <--gar-out>")
  parser.add_argument("--gar-rule-args", dest="rule_args", nargs="*", default=None, metavar="KEY:VALUE",
                      help="`--aggregator-args` of every rule of --gar-rules (e.g. iterations:1 nu:1e-6 for geometric-median)")
  parser.add_argument("--gar-worker-momentum", dest="worker_momentum", type=float, default=None, metavar="BETA",
                      help="also time the worker-momentum kernel with this beta on the [w, d] rows of a rank")
  args = parser.parse_args()
  world = int(os.environ.get("WORLD_SIZE", "1"))
  rank = int(os.environ.get("RANK", "0"))
  local = int(os.environ.get("LOCAL_RANK", "0"))
  device = torch.device("cuda", local)
  torch.cuda.set_device(device)
  if world > 1:
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=device)
  if rank != 0:
    tools.set_rank_tag("r" + str(rank))
  n = args.nb_workers
  # measured peer bandwidth of this box: every rank pulls 256 MiB from its right neighbour at the same time (kernel P2P loads), the
  # denominator of the link-roofline fractions below
  peer_gbs = None
  if world > 1:
    import ctypes
    from aggregathor_b200 import native
    from aggregathor_b200.parallel.symm import SymmetricHeap
    nbytes = 256 << 20
    heap = SymmetricHeap(SymmetricHeap.required(nbytes), device)
    heap.region("buf", nbytes)
    dst = torch.empty(nbytes // 4, dtype=torch.float32, device=device)
    comm = native.library("op_comm")
    src = heap.peer((rank + 1) % world, "buf")
    times = []
    for it in range(6):
      torch.cuda.synchronize()
      dist.barrier()
      torch.cuda.synchronize()
      begin, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      begin.record()
      comm.agb_comm_p2p_copy(ctypes.c_ulonglong(src), ctypes.c_ulonglong(dst.data_ptr()), ctypes.c_longlong(nbytes // 4), ctypes.c_int(0), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
      end.record()
      torch.cuda.synchronize()
      ms = torch.tensor([begin.elapsed_time(end)], device=device, dtype=torch.float64)
      dist.all_reduce(ms, op=dist.ReduceOp.MAX)
      if it >= 2:
        times.append(float(ms.item()))
    peer_gbs = nbytes / min(times) / 1e6
    if rank == 0:
      print("measured peer pull bandwidth: %.1f GB/s per GPU (all ranks pulling at once)" % peer_gbs)
    del heap, dst
  layout = FlatLayout()
  layout.add("theta", (args.d,))
  layout.freeze()
  d = layout.padded_size
  w = n // world
  results = {}
  for rule in args.rules.split(","):
    f = args.byz if args.byz is not None else 1 if rule == "bulyan" and n < 11 else 2
    name = {"krum": "krum", "bulyan": "bulyan"}.get(rule, rule)
    gar = aggregators.instantiate(name, n, f, args.rule_args or [])
    sgd = build(optimizers, "optimizer", "sgd", [])
    fused = FusedAggregation(gar, layout, n, sgd, device=device, keep_aggregate=True)
    base = BaselineAggregation(gar, layout, n, build(optimizers, "optimizer", "sgd", []), device=device)
    gen = torch.Generator(device=device).manual_seed(1234)
    init = torch.randn(d, device=device, generator=gen)
    fused.params.copy_(init)
    base.params.copy_(init)
    grads = torch.empty((w, d), device=device)
    for j in range(w):
      g = torch.Generator(device=device).manual_seed(100 + rank * w + j)
      grads[j].normal_(0.0, 1.0, generator=g)
      if rank * w + j >= n - f:
        grads[j].mul_(20.0).add_(3.0)  # the last f workers are outliers
    fused.grads.copy_(grads)
    base.grads.copy_(grads)
    attack = attacks.instantiate(args.attack, n, f, []) if args.attack else None
    byz_slots = list(range(n - f, n))

    def craft(engine):
      if attack is not None:
        engine.craft_byzantine(byz_slots, attack.mode, attack.coef)

    torch.cuda.synchronize()
    if world > 1:
      dist.barrier()
    craft(fused)
    fused.step(0.1)
    craft(base)
    base.step(0.1)
    torch.cuda.synchronize()
    if attack is not None and args.dump_rows and rank == world - 1:
      rows = fused.visible_rows()
      os.makedirs(args.out, exist_ok=True)
      torch.save({"rows": torch.stack([rows[i].cpu() for i in range(n)]), "byzantine": byz_slots, "mode": attack.mode, "coef": attack.coef},
                 os.path.join(args.out, "gar_rows_%s_%d.pt" % (rule, world)))
    diff = float((fused.params - base.params).abs().max())
    digest = gar_ops.checksum(fused.params)
    digests = [torch.zeros_like(digest) for _ in range(world)]
    if world > 1:
      dist.all_gather(digests, digest)
    else:
      digests = [digest]
    identical = len({int(x.item()) for x in digests}) == 1

    def time_engine(engine):
      torch.cuda.synchronize()
      if world > 1:
        dist.barrier()
      torch.cuda.synchronize()
      begin, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      begin.record()
      for _ in range(args.iters):
        craft(engine)
        engine.step(0.1)
      end.record()
      torch.cuda.synchronize()
      ms = torch.tensor([begin.elapsed_time(end) / args.iters], device=device, dtype=torch.float64)
      if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
      return float(ms.item())

    for engine in (fused, base):
      for _ in range(3):
        craft(engine)
        engine.step(0.1)
    fused_ms = time_engine(fused)
    base_ms = time_engine(base)
    attack_entry = {}
    if attack is not None:
      def time_craft(fn):
        for _ in range(3):
          fn()
        torch.cuda.synchronize()
        if world > 1:
          dist.barrier()
        torch.cuda.synchronize()
        begin, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        begin.record()
        for _ in range(args.iters):
          fn()
        end.record()
        torch.cuda.synchronize()
        ms = torch.tensor([begin.elapsed_time(end) / args.iters], device=device, dtype=torch.float64)
        if world > 1:
          dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms.item())
      craft_ms = time_craft(lambda: fused.craft_byzantine(byz_slots, attack.mode, attack.coef))
      # the torch reference on this device, over the full [n, d] matrix (what a torch attack would run after an all-gather)
      reference_ms = time_craft(lambda: _ops.torch_craft_byzantine_(base._gathered, byz_slots, attack.mode, attack.coef))
      craft_bytes = n * d * 4   # (H + k) * d * 4: every honest value read once, every Byzantine value written once (over all ranks)
      attack_entry = {"attack": attack.mode, "coef": attack.coef, "k": f, "craft_ms": craft_ms, "torch_reference_ms": reference_ms,
                      "craft_bytes": craft_bytes, "craft_gbs": craft_bytes / craft_ms / 1e6,
                      "torch_reference_gbs": craft_bytes / reference_ms / 1e6}
    # overlapped variant (Krum / Bulyan): the distance pass of the first three buckets runs as separate small launches (in training:
    # on a side stream under the backward pass); what stays exposed at the end of the step is the finish kernel alone
    exposed_ms = bucketed_ms = None
    if rule in ("krum", "bulyan", "mda"):
      c1, c2, c3 = (d // 2) // 8 * 8, (d // 5) // 8 * 8, (d // 16) // 8 * 8
      over = FusedAggregation(gar, layout, n, build(optimizers, "optimizer", "sgd", []), device=device, keep_aggregate=True,
                              buckets=[(c1, d), (c2, c1), (c3, c2), (0, c3)], device_state=True)
      over.params.copy_(init)
      over.grads.copy_(grads)
      side = torch.cuda.Stream(device=device, priority=-1)

      def over_step(time_finish=None):
        over.prepare(0.1)
        side.wait_stream(torch.cuda.current_stream())
        for k in range(3):
          over.phase_a(k, stream=side)
        torch.cuda.current_stream().wait_stream(side)
        if time_finish is not None:
          time_finish[0].record()
        over.step(prepared=True)
        if time_finish is not None:
          time_finish[1].record()
      over_step()
      torch.cuda.synchronize()
      over_diff = float((over.params - base.params).abs().max()) if False else None
      for _ in range(3):
        over_step()
      torch.cuda.synchronize()
      if world > 1:
        dist.barrier()
      torch.cuda.synchronize()
      total_b, total_e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      pairs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.iters)]
      total_b.record()
      for it in range(args.iters):
        over_step(pairs[it])
      total_e.record()
      torch.cuda.synchronize()
      ms = torch.tensor([total_b.elapsed_time(total_e) / args.iters, sum(b.elapsed_time(e) for b, e in pairs) / args.iters], device=device, dtype=torch.float64)
      if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
      bucketed_ms, exposed_ms = float(ms[0]), float(ms[1])
      del over
    slice_bytes = (fused.hi - fused.lo) * 4
    # bytes entering each GPU over NVLink: slices of the (n - w) remote workers + the (R-1)/R of the parameters pushed by peers
    nvlink_in = (n - w) * slice_bytes + (d * 4 - slice_bytes) if world > 1 else 0
    hbm = n * slice_bytes + 2 * slice_bytes
    results[rule] = {"f": f, "fused_ms": fused_ms, "baseline_ms": base_ms, "speedup": base_ms / fused_ms, "max_abs_diff_vs_baseline": diff,
                     "replicas_identical": identical, "nvlink_bytes_in_per_gpu": nvlink_in, "gather_gbs_per_gpu": (n * slice_bytes) / fused_ms / 1e6,
                     "nvlink_gbs_per_gpu": nvlink_in / fused_ms / 1e6 if world > 1 else None,
                     "measured_peer_gbs": peer_gbs, "frac_of_measured_peer": (nvlink_in / fused_ms / 1e6) / peer_gbs if peer_gbs else None,
                     "bucketed_total_ms": bucketed_ms, "finish_kernel_exposed_ms": exposed_ms,
                     "local_hbm_bytes": hbm, "hbm_gbs": hbm / fused_ms / 1e6 if world == 1 else None}
    results[rule].update(attack_entry)
    if args.rule_args is not None:
      results[rule]["rule_args"] = args.rule_args
    if rule in ("geometric-median", "centered-clipping"):
      # T + 1 passes, each reading the n rows of the owned coordinates once (the first from the peers, the others from the staged copy)
      spec = gar.fused_spec()
      passes_bytes = (spec.iterations + 1) * n * slice_bytes
      radius = {"nu": spec.nu} if rule == "geometric-median" else {"tau": spec.tau}
      results[rule].update({"iterations": spec.iterations, **radius, "pass_bytes": passes_bytes, "pass_gbs": passes_bytes / fused_ms / 1e6})
    if rank == 0:
      print(rule, json.dumps(results[rule]))
    del fused, base
    torch.cuda.empty_cache()
  report = {"world": world, "n": n, "d": args.d, "results": results}
  if args.worker_momentum is not None:
    beta, c = _ops.check_worker_momentum(args.worker_momentum, 0.0)
    rows = torch.randn((w, d), device=device)
    momenta = torch.zeros((w, d), device=device)
    for _ in range(3):
      gar_ops.worker_momentum_(rows, momenta, beta, c)
    torch.cuda.synchronize()
    if world > 1:
      dist.barrier()
    begin, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    begin.record()
    for _ in range(args.iters):
      gar_ops.worker_momentum_(rows, momenta, beta, c)
    end.record()
    torch.cuda.synchronize()
    ms = torch.tensor([begin.elapsed_time(end) / args.iters], device=device, dtype=torch.float64)
    if world > 1:
      dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    momentum_bytes = 16 * w * d   # G and M of every element read and written once
    report["worker_momentum"] = {"beta": beta, "w": w, "d": d, "ms": float(ms.item()), "bytes": momentum_bytes,
                                 "gbs": momentum_bytes / float(ms.item()) / 1e6}
    if rank == 0:
      print("worker-momentum", json.dumps(report["worker_momentum"]))
    del rows, momenta
  if rank == 0:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "gar_bench_%d.json" % world), "w") as fd:
      json.dump(report, fd, indent=1)
  if world > 1:
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
  main()

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
`--gar-attack min-max|min-sum` (Shejwalkar & Houmansadr, NDSS 2021; `--gar-attack-args deviation:unit-vec|sign|std`) also reports the
gamma every rank solved, and times the crafting kernel alternated round by round with ALIE's on the same rows.
`--gar-attack mimic` (Karimireddy, He & Jaggi, ICLR 2022; `--gar-attack-args warmup:<T0>`) reports the target i* every rank chose and
whether the Byzantine rows equal the baseline engine's, and times the warm-up kernel and the copy pass, each alternated with ALIE.
`--gar-attack fang-krum|fang-trim` (Fang, Cao, Jia & Gong, USENIX Security 2020; `--gar-attack-args threshold:<x>` or `scale:<beta>
seed:<int>`) times the crafting kernel alternated round by round with ALIE's on the same rows. fang-krum also reports the gamma, the
candidate t and the selected flag every rank solved, and times the same kernel without its candidate search (`nosearch_*`: the passes
alone, so `search_share_ms` is the search's own cost); fang-trim reports whether the Byzantine rows equal the baseline engine's.
`--gar-rule-args key:value ...` passes the same `--aggregator-args` to every rule (rules ignore keys they do not use). The
`geometric-median` and `centered-clipping` entries also report their T + 1 passes' (T + 1) * n * slice * 4 bytes and their rate.
`--gar-worker-momentum beta` also times the worker-momentum kernel alone on the [w, d] rows of a rank (`ops.gar.worker_momentum_`,
dampening 0), with the 16 * w * d bytes it must move (G and M read and written once).
`--gar-pre-aggregation nnm` runs both engines with nearest-neighbour mixing before every rule (the checks above then hold for the
mixed step), and also times the fused step of each rule without NNM, alternating with and without in the same process, to report
the measured cost of the mix (`nnm_ms`, `plain_ms`, `nnm_overhead_ms`: medians over the alternated rounds).
`--gar-pre-aggregation arc` (adaptive robust clipping) and `arc+nnm` (ARC, then NNM) do the same, with keys `arc_ms`,
`arc_overhead_ms` and `arc_nnm_ms`, `arc_nnm_overhead_ms`.
`--gar-pre-aggregation bucketing --gar-bucket-size s` builds every rule for the n' = ceil(n / s) bucket means and compares it with the
same rule on the n plain rows (`bucketing_ms`, `plain_ms`, `bucketing_overhead_ms`, `rule_rows`); a rule that refuses the n rows
(e.g. SMEA at (32, 4)) is timed with bucketing only (`plain_refused`).
`dnc` (divide-and-conquer) takes `--gar-rule-args iterations:<T> subsample:<b> c:<c> seed:<s>`; both engines draw the same samples (the
step key is the update count), so the fused-vs-baseline check holds for it as for the other rules; its entry also reports the rows
each engine kept in the checked step (`fused_mask`, `baseline_mask`, `masks_agree`).
`fltrust` seeds a synthetic root gradient on rank 0, which the fused kernel reads over P2P and the baseline engine broadcasts; the
fused-vs-baseline check holds for it as for the other rules.
`foolsgold` updates the per-worker histories at every step (both engines start from zero histories and take the same steps); its
entry reports the rows of non-zero weight (`weighted_rows`), the largest difference between the two engines' histories after the
checked step, and the local HBM bytes of one fused step counted from the shapes (`foolsgold_hbm_bytes`: the history pass reads g and H
and writes H, re-reads the histories of the 8-row blocks it pairs when n > 8 and stores the staged rows when there is a tile; phase D
reads the weighted rows; the SGD update reads and writes the parameters and stores the kept aggregate) with the rate they imply.
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


def foolsgold_hbm_bytes(n, slice_bytes, weighted, staged):
  """Local HBM bytes of one fused FoolsGold step over `slice_bytes` owned bytes per row (see the module docstring)."""
  size = [min(8, n - 8 * b) for b in range(-(-n // 8))]   # the rows of every 8-row block
  rereads = sum(size[1:]) + sum(size[bi] + (size[bj] if bi > 0 else 0) for bi in range(len(size)) for bj in range(bi + 1, len(size)))
  return (3 * n + rereads + (n if staged else 0) + weighted + 3) * slice_bytes


def main():
  parser = argparse.ArgumentParser()
  parser.add_argument("--gar-dim", dest="d", type=int, default=25557032)
  parser.add_argument("--gar-workers", dest="nb_workers", type=int, default=8)
  parser.add_argument("--gar-iters", dest="iters", type=int, default=10)
  parser.add_argument("--gar-rules", dest="rules", type=str, default="average,average-nan,median,averaged-median,krum,bulyan")
  parser.add_argument("--gar-out", dest="out", type=str, default=".")
  parser.add_argument("--gar-byz", dest="byz", type=int, default=None, help="declared Byzantine workers f of every rule (default: 1 for Bulyan below 11 workers, else 2)")
  parser.add_argument("--gar-attack", dest="attack", choices=("alie", "ipm", "min-max", "min-sum", "mimic", "fang-krum", "fang-trim"), default=None,
                      help="omniscient attack by the last f workers, crafted every step")
  parser.add_argument("--gar-attack-args", dest="attack_args", nargs="*", default=None, metavar="KEY:VALUE",
                      help="`--attack-args` of --gar-attack (e.g. deviation:std for min-max / min-sum)")
  parser.add_argument("--gar-dump-rows", dest="dump_rows", action="store_true", help="with --gar-attack: save the last rank's view of every row to <--gar-out>")
  parser.add_argument("--gar-rule-args", dest="rule_args", nargs="*", default=None, metavar="KEY:VALUE",
                      help="`--aggregator-args` of every rule of --gar-rules (e.g. iterations:1 nu:1e-6 for geometric-median)")
  parser.add_argument("--gar-worker-momentum", dest="worker_momentum", type=float, default=None, metavar="BETA",
                      help="also time the worker-momentum kernel with this beta on the [w, d] rows of a rank")
  parser.add_argument("--gar-pre-aggregation", dest="pre_aggregation", choices=("none", "nnm", "arc", "arc+nnm", "bucketing"), default="none",
                      help="pre-aggregation of both engines, with the rule's f (nnm: nearest-neighbour mixing, arc: adaptive robust clipping, "
                           "arc+nnm: both; bucketing: means of buckets of --gar-bucket-size rows, the rule built for ceil(n / s) rows); "
                           "also times each rule without it")
  parser.add_argument("--gar-bucket-size", dest="bucket_size", type=int, default=2, help="rows per bucket s of --gar-pre-aggregation bucketing")
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
  bucketing = args.pre_aggregation == "bucketing"
  rows = -(-n // args.bucket_size) if bucketing else n   # the rows every rule sees
  for rule in args.rules.split(","):
    f = args.byz if args.byz is not None else 1 if rule == "bulyan" and rows < 11 else 2
    name = {"krum": "krum", "bulyan": "bulyan"}.get(rule, rule)
    gar = aggregators.instantiate(name, rows, f, args.rule_args or [])
    sgd = build(optimizers, "optimizer", "sgd", [])
    mix = dict(pre_aggregation=args.pre_aggregation, nb_decl_byz=f)
    if bucketing:
      mix.update(bucket_size=args.bucket_size, bucketing_seed=0)
    fused = FusedAggregation(gar, layout, n, sgd, device=device, keep_aggregate=True, **mix)
    base = BaselineAggregation(gar, layout, n, build(optimizers, "optimizer", "sgd", []), device=device, **mix)
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
    if fused.root is not None and rank == 0:   # FLTrust: a synthetic root gradient, on rank 0 only (the engines take it from there)
      root = torch.empty(d, device=device).normal_(0.0, 1.0, generator=torch.Generator(device=device).manual_seed(99))
      fused.root.copy_(root)
      base.root.copy_(root)
    attack = attacks.instantiate(args.attack, n, f, args.attack_args or []) if args.attack else None
    byz_slots = list(range(n - f, n))
    extra = {"deviation": attack.deviation} if attack is not None and attack.deviation is not None else {}
    mimic = attack is not None and attack.mode == "mimic"
    if mimic:
      extra = {"warmup": attack.warmup}
    fang = attack.mode if attack is not None and attack.mode in _ops.FANG_MODES else None
    if fang:
      extra = {key: getattr(attack, key) for key in ("threshold", "scale", "seed") if getattr(attack, key) is not None}

    def craft(engine):
      if attack is not None:
        engine.craft_byzantine(byz_slots, attack.mode, attack.coef, **extra)

    torch.cuda.synchronize()
    if world > 1:
      dist.barrier()
    craft(fused)
    fused.step(0.1)
    craft(base)
    base.step(0.1)
    torch.cuda.synchronize()
    mask_entry = {}
    if rule == "dnc":   # the rows each engine kept in the checked step (bit i: row i)
      fused_mask = int(fused.launcher.info[1].item()) & 0xffffffff
      base_mask = int(gar_ops._launcher(base._gathered.device, n, rows).info[1].item()) & 0xffffffff
      mask_entry = {"fused_mask": fused_mask, "baseline_mask": base_mask, "masks_agree": fused_mask == base_mask}
    if rule == "fltrust":   # the rows of non-zero weight, the only ones the weighted sum reads
      coefs = fused.launcher.fltrust_out[2 * gar_ops.MAX_WORKERS + 1:2 * gar_ops.MAX_WORKERS + 1 + n].cpu()
      mask_entry = {"weighted_rows": int((coefs != 0).sum())}
    if rule == "foolsgold":   # the rows phase D reads, and the histories after the checked step against the baseline engine's
      at = gar_ops.FOOLSGOLD_SUMS + gar_ops.MAX_WORKERS
      coefs = fused.launcher.foolsgold_out[at:at + n].cpu()
      mask_entry = {"weighted_rows": int((coefs != 0).sum()), "history_max_abs_diff_vs_baseline": float((fused.full_history() - base.history).abs().max())}
    gamma_entry = {}
    if attack is not None and attack.deviation is not None:
      # gamma as every rank solved it (fused engine), and as the baseline engine's stand-alone kernel solved it on the gathered rows
      gamma = torch.tensor([fused.last_craft[0]], dtype=torch.float32, device=device)
      gammas = [torch.zeros_like(gamma) for _ in range(world)]
      if world > 1:
        dist.all_gather(gammas, gamma)
      else:
        gammas = [gamma]
      gamma_entry = {"deviation": attack.deviation, "gamma_per_rank": [float(x.item()) for x in gammas], "baseline_gamma": base.last_craft[0]}
    if mimic:
      # i* as every rank chose it (fused engine) and as the baseline engine's stand-alone kernel chose it on the gathered rows; the
      # Byzantine rows this rank sees through the peer mapping against the baseline engine's gathered matrix, bit for bit
      target = fused.attack_state["istar"].to(torch.int64)
      targets = [torch.zeros_like(target) for _ in range(world)]
      if world > 1:
        dist.all_gather(targets, target)
      else:
        targets = [target]
      rows = fused.visible_rows()
      same = torch.tensor([int(all(torch.equal(rows[b].view(torch.int32), base._gathered[b].view(torch.int32)) for b in byz_slots))], device=device)
      if world > 1:
        dist.all_reduce(same, op=dist.ReduceOp.MIN)
      gamma_entry = {"warmup": attack.warmup, "istar_per_rank": [int(x.item()) for x in targets], "baseline_istar": int(base.attack_state["istar"][0]),
                     "rows_match_baseline": bool(same.item())}
    if fang == "fang-krum":
      # gamma, t and the selected flag as every rank solved them (fused engine), and the baseline engine's on the gathered rows
      solved = torch.tensor([fused.last_craft[0], fused.last_craft[2], float(fused.last_craft[1])], dtype=torch.float64, device=device)
      solved_all = [torch.zeros_like(solved) for _ in range(world)]
      if world > 1:
        dist.all_gather(solved_all, solved)
      else:
        solved_all = [solved]
      gamma_entry = {"gamma_per_rank": [float(x[0]) for x in solved_all], "t_per_rank": [int(x[1]) for x in solved_all],
                     "selected_per_rank": [bool(x[2]) for x in solved_all], "gamma_max": fused.last_craft[3], "baseline_gamma": base.last_craft[0],
                     "baseline_t": base.last_craft[2], "baseline_selected": base.last_craft[1]}
    if fang == "fang-trim":
      # the Byzantine rows this rank sees through the peer mapping against the baseline engine's gathered matrix, bit for bit
      rows = fused.visible_rows()
      same = torch.tensor([int(all(torch.equal(rows[b].view(torch.int32), base._gathered[b].view(torch.int32)) for b in byz_slots))], device=device)
      if world > 1:
        dist.all_reduce(same, op=dist.ReduceOp.MIN)
      gamma_entry = {"rows_match_baseline": bool(same.item())}
    if attack is not None and args.dump_rows and rank == world - 1:
      rows = fused.visible_rows()
      os.makedirs(args.out, exist_ok=True)
      gamma = fused.last_craft[0] if attack.deviation is not None or fang == "fang-krum" else None
      torch.save({"rows": torch.stack([rows[i].cpu() for i in range(n)]), "byzantine": byz_slots, "mode": attack.mode, "coef": attack.coef,
                  "deviation": attack.deviation, "gamma": gamma},
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
    mix_entry = {}
    if fused.mix is not None:
      # the same rule without the pre-aggregation on the same rows, alternated with the pre-aggregating engine round by round (clock and
      # thermal drift hit both); keys are prefixed by the pre-aggregation: nnm_ms, arc_ms, arc_nnm_ms, ...
      # with bucketing the plain arm is the same rule built for the n rows, which it may refuse (e.g. SMEA at (32, 4)): then only
      # the bucketing arm is timed
      try:
        plain_gar = aggregators.instantiate(name, n, f, args.rule_args or []) if bucketing else gar
        plain = FusedAggregation(plain_gar, layout, n, build(optimizers, "optimizer", "sgd", []), device=device, keep_aggregate=True)
      except tools.UserException as err:
        plain, plain_refused = None, str(err)
      if plain is not None:
        plain.params.copy_(init)
        plain.grads.copy_(fused.grads)
        for _ in range(3):
          craft(plain)
          plain.step(0.1)
      rounds = {"pre": [], "plain": []}
      for _ in range(5):
        rounds["pre"].append(time_engine(fused))
        if plain is not None:
          rounds["plain"].append(time_engine(plain))
      median = lambda values: sorted(values)[len(values) // 2] if values else None
      pre_ms, plain_ms = median(rounds["pre"]), median(rounds["plain"])
      key = fused.mix.replace("+", "_")
      # bucketing stages only the rule's rows (its n' means), the other pre-aggregations all n rows
      slice_rows = fused.spec.n * (fused.hi - fused.lo) * 4
      # local HBM bytes of the staged tile: the staging store; ARC's clip pass (read + write of its k rows); NNM's mix pass (read + write)
      # after its distance pass (a read of the tile when ARC staged it); the rule's read of the tile; and one more read for the distance
      # pass of the pre-aggregated rows (Krum / Bulyan / MDA / SMEA)
      k = _ops.arc_clip_count(n, f) if "arc" in fused.mix else 0
      tile_reads = 2 + (1 if rule in ("krum", "bulyan", "mda", "smea") else 0) + (2 if "nnm" in fused.mix else 0) + (1 if fused.mix == "arc+nnm" else 0)
      mix_entry = {"pre_aggregation": fused.mix, key + "_ms": pre_ms, "plain_ms": plain_ms,
                   key + "_overhead_ms": pre_ms - plain_ms if plain_ms is not None else None,
                   key + "_rounds_ms": rounds["pre"], "plain_rounds_ms": rounds["plain"],
                   key + "_tile_hbm_bytes": tile_reads * slice_rows + 2 * k * (fused.hi - fused.lo) * 4}
      if k:
        mix_entry["arc_clipped_rows"] = k
      if bucketing:
        mix_entry.update(bucket_size=args.bucket_size, rule_rows=rows)
        if plain is None:
          mix_entry["plain_refused"] = plain_refused
      del plain
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
      def craft_at(engine, t):
        """Mimic at warm-up step t (t < T0: the warm-up kernel; t = T0: the copy pass); other attacks: their usual crafting."""
        if mimic:
          engine.attack_state["t"] = t
        engine.craft_byzantine(byz_slots, attack.mode, attack.coef, **extra)
      craft_ms = time_craft(lambda: craft_at(fused, 1))
      # the torch reference on this device, over the full [n, d] matrix (what a torch attack would run after an all-gather)
      if mimic:
        ref_state = _ops.mimic_state(base._gathered.shape[1], device)

        def reference():
          ref_state["t"] = 1
          _ops.torch_mimic_step_(base._gathered, byz_slots, ref_state, attack.warmup)
        reference_ms = time_craft(reference)
      else:
        ref_extra = dict(extra, f=f) if fang == "fang-krum" else dict(extra, step=1) if fang == "fang-trim" else extra
        reference_ms = time_craft(lambda: _ops.torch_craft_byzantine_(base._gathered, byz_slots, attack.mode, attack.coef, **ref_extra))
      craft_bytes = n * d * 4   # (H + k) * d * 4: every honest value read once, every Byzantine value written once (over all ranks)
      if attack.deviation is not None:
        # Min-Max / Min-Sum read the honest values again in the write pass, and Min-Max once more in its honest-distance pass
        craft_bytes += (2 if attack.mode == "min-max" else 1) * (n - f) * d * 4
      if fang == "fang-krum":
        # the honest values are read by the statistics pass, the honest distance pass and the write pass (Min-Max's bytes)
        craft_bytes += 2 * (n - f) * d * 4
      if mimic:
        # warm-up: the honest rows read in passes 1 and 2 (twice in pass 2 beyond the registers, counted once), z read twice and written
        # once, y written and read, then h_{i*} read and the k rows written; the copy pass alone: h_{i*} read, the k rows written
        craft_bytes = (2 * (n - f) + 5 + 1 + f) * d * 4
        copy_bytes = (1 + f) * d * 4
      attack_entry = {"attack": attack.mode, "coef": attack.coef, "k": f, "craft_ms": craft_ms, "torch_reference_ms": reference_ms,
                      "craft_bytes": craft_bytes, "craft_gbs": craft_bytes / craft_ms / 1e6,
                      "torch_reference_gbs": craft_bytes / reference_ms / 1e6}
      attack_entry.update(gamma_entry)
      if mimic:
        # the warm-up kernel and the copy pass, each alternated round by round with ALIE's kernel on the same rows
        alie = attacks.instantiate("alie", n, f, [])
        rounds = {"warmup": [], "copy": [], "alie": []}
        for _ in range(5):
          rounds["warmup"].append(time_craft(lambda: craft_at(fused, 1)))
          rounds["copy"].append(time_craft(lambda: craft_at(fused, attack.warmup)))
          rounds["alie"].append(time_craft(lambda: fused.craft_byzantine(byz_slots, "alie", alie.coef)))
        median = lambda values: sorted(values)[len(values) // 2]
        attack_entry.update({"warmup_rounds_ms": rounds["warmup"], "copy_rounds_ms": rounds["copy"], "alie_craft_rounds_ms": rounds["alie"],
                             "warmup_median_ms": median(rounds["warmup"]), "copy_median_ms": median(rounds["copy"]),
                             "alie_craft_median_ms": median(rounds["alie"]), "warmup_bytes": craft_bytes, "copy_bytes": copy_bytes,
                             "warmup_gbs": craft_bytes / median(rounds["warmup"]) / 1e6, "copy_gbs": copy_bytes / median(rounds["copy"]) / 1e6})
      if attack.deviation is not None or fang:
        # ALIE's crafting kernel on the same rows, alternated with this attack's round by round (clock and thermal drift hit both).
        # Repeated calls at one step's epoch pass the flag barriers at once: with R > 1 they time the kernels, their gamma is not checked.
        alie = attacks.instantiate("alie", n, f, [])
        rounds = {"craft": [], "alie": [], "nosearch": []}
        honest = [i for i in range(n) if i not in byz_slots]

        def nosearch():
          """fang-krum's kernel with the candidate search skipped (gamma = gamma_max): the statistics, exchange and write passes alone."""
          gar_ops.craft(fused._rows, fused.segments, honest, byz_slots, "fang-krum", None, f=fused.f, threshold=attack.threshold,
                        launcher=fused.launcher, mailboxes=fused._mailboxes, R=world, rank=rank, signals=fused._signals, epoch=fused.epoch + 1,
                        epoch_ptr=fused.epoch_dev, search=False)
        for _ in range(5):
          rounds["craft"].append(time_craft(lambda: fused.craft_byzantine(byz_slots, attack.mode, attack.coef, **extra)))
          rounds["alie"].append(time_craft(lambda: fused.craft_byzantine(byz_slots, "alie", alie.coef)))
          if fang == "fang-krum":
            rounds["nosearch"].append(time_craft(nosearch))
        median = lambda values: sorted(values)[len(values) // 2]
        attack_entry.update({"craft_rounds_ms": rounds["craft"], "alie_craft_rounds_ms": rounds["alie"], "craft_median_ms": median(rounds["craft"]),
                             "alie_craft_median_ms": median(rounds["alie"]), "craft_median_gbs": craft_bytes / median(rounds["craft"]) / 1e6})
        if fang == "fang-krum":
          attack_entry.update({"nosearch_rounds_ms": rounds["nosearch"], "nosearch_median_ms": median(rounds["nosearch"]),
                               "search_share_ms": median(rounds["craft"]) - median(rounds["nosearch"])})
    # overlapped variant (Krum / Bulyan): the distance pass of the first three buckets runs as separate small launches (in training:
    # on a side stream under the backward pass); what stays exposed at the end of the step is the finish kernel alone
    exposed_ms = bucketed_ms = None
    if rule in ("krum", "bulyan", "mda", "smea") and fused.mix is None:   # no bucketed distance pass with NNM
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
    results[rule].update(mix_entry)
    results[rule].update(mask_entry)
    if rule == "foolsgold":
      counted = foolsgold_hbm_bytes(n, slice_bytes, mask_entry["weighted_rows"], fused.staging is not None)
      results[rule].update(foolsgold_hbm_bytes=counted, foolsgold_hbm_gbs=counted / fused_ms / 1e6)
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
  report = {"world": world, "n": n, "d": args.d, "pre_aggregation": args.pre_aggregation, "results": results}
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

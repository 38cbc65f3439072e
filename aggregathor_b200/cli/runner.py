"""Main training driver (reference: `runner.py:1-610`).

Same phases, same flags, same log/eval/checkpoint formats; SPMD instead of in-graph replication: launched once per
GPU (`torchrun`/`deploy.py`) or as a single process hosting every logical worker on one device. The rank that holds
`ps:0` (rank 0) prints, evaluates, checkpoints and writes summaries; the other ranks stay quiet.
"""

import argparse
import math
import os
import pathlib
import signal
import sys
import threading
import time

import torch
import torch.distributed as dist

from .. import aggregators, attacks, cluster, config, experiments, tools
from ..engine import services
from ..engine.trainer import Manager

exit_pending = False


def mark_exit(*args, **kwargs):
  global exit_pending
  exit_pending = True


def make_parser():
  parser = argparse.ArgumentParser(description="Start/continue a distributed training session.", formatter_class=argparse.RawTextHelpFormatter)
  add = parser.add_argument
  add("--client", type=str, default="", help="Trusted node URL in the cluster (usually the parameter server) to connect to as a client; one and only one of '--server' and '--client' must be specified")
  add("--server", type=str, default="", help="Full JSON cluster specification, on which to act as the only parameter server, or special value(s): " + tools.cluster_parsers + "; one and only one of '--server' and '--client' must be specified")
  add("--ps-job-name", type=str, default=config.default_ps_job_name, help="Parameter server job name")
  add("--ev-job-name", type=str, default=config.default_ev_job_name, help="Evaluation job name (may be the parameter server job name)")
  add("--wk-job-name", type=str, default=config.default_wk_job_name, help="Worker job name")
  add("--experiment", type=str, required=True, help="Experiment to run on the cluster")
  add("--experiment-args", nargs="*", help="Additional arguments to pass to the underlying experiment")
  add("--aggregator", type=str, required=True, help="Gradient aggregation rule to use")
  add("--aggregator-args", nargs="*", help="Additional arguments to pass to the underlying GAR")
  add("--optimizer", type=str, default="sgd", help="Optimizer to use")
  add("--optimizer-args", nargs="*", help="Additional arguments to pass to the underlying optimizer")
  add("--learning-rate", type=str, default="fixed", help="Type of learning rate decay to use")
  add("--learning-rate-args", nargs="*", help="Additional arguments to pass to the underlying learning rate")
  add("--l1-regularize", type=float, default=-1., help="l1 regularization strength to use, non-positive for none, non-positive by default")
  add("--l2-regularize", type=float, default=-1., help="l2 regularization strength to use, non-positive for none, non-positive by default")
  add("--nb-workers", type=int, required=True, help="Total number of workers")
  add("--nb-decl-byz-workers", type=int, default=0, help="Number of declared Byzantine workers (i.e. value of 'f')")
  add("--nb-real-byz-workers", type=int, default=0, help="Number of real Byzantine workers")
  add("--attack", type=str, default="", help="Attack to use (ignored if --nb-real-byz-workers is 0)")
  add("--attack-args", nargs="*", help="Additional arguments to pass to the underlying attack (ignored if --nb-real-byz-workers is 0)")
  add("--max-step", "--max-steps", dest="max_step", type=int, default=config.default_max_step, help="Number of additional steps to perform before stopping the training, non-positive for no limit")
  add("--checkpoint-dir", type=str, default="", help="Checkpoint directory to use, will be created if inexistent")
  add("--checkpoint-delta", type=int, default=config.default_checkpoint_delta, help="Save checkpoint after the given step delta, negative for unused")
  add("--checkpoint-period", type=float, default=config.default_checkpoint_period, help="Save checkpoint at least every given period (in s), negative for unused")
  add("--summary-dir", type=str, default="", help="Summary directory to use, '-' for none, defaults to '--checkpoint-dir'")
  add("--summary-delta", type=float, default=config.default_summary_delta, help="Save summaries after the given step delta, negative for unused")
  add("--summary-period", type=float, default=config.default_summary_period, help="Save summaries at least every given period (in s), negative for unused")
  add("--evaluation-file", type=str, default="", help="File in which to write the accuracy evaluations (format: wall time (in s)<tab>global step<tab>name:value<tab>...), '-' for none, defaults to '<checkpoint dir>/" + config.default_evaluation_file_name + "'")
  add("--evaluation-delta", type=int, default=config.default_evaluation_delta, help="Evaluate the model after the given step delta, negative for unused")
  add("--evaluation-period", type=float, default=config.default_evaluation_period, help="Evaluate the model at least every given period (in s), negative for unused")
  add("--use-gpu", action="store_true", default=False, help="Use target GPU devices if available")
  add("--reuse-gpu", action="store_true", default=False, help="Allow target GPU devices to be used by several entities, implies '--use-gpu'")
  add("--use-tpu", action="store_true", default=False, help="Use target TPU devices if available (accepted for compatibility: there is no TPU path)")
  add("--reuse-tpu", action="store_true", default=False, help="Allow target TPU devices to be used by several entities, implies '--use-tpu'")
  add("--no-wait", action="store_true", default=False, help="Do not wait for a signal before exiting when acting as a server")
  add("--trace", action="store_true", default=False, help="Print a (performance) debugging message for every important step of the graph execution")
  add("--stdout-to", type=str, default="-", help="Redirect the standard output to the given file (overwritten if exists), '-' for none, '-' by default")
  add("--stderr-to", type=str, default="-", help="Redirect the standard error output to the given file (overwritten if exists), '-' for none, '-' by default")
  add("--MPI", action="store_true", default=False, help="Accepted for compatibility (the reference's grpc+mpi transport); ranks always talk over NVLink/NCCL or gloo")
  # Additions
  add("--engine", type=str, default="auto", choices=("auto", "fused", "baseline", "host"), help="Aggregation engine: fused sm_90a kernel over peer memory, NCCL all-gather baseline, or host C++")
  add("--nn-backend", type=str, default="auto", choices=("auto", "native", "torch"), help="Provider of the model kernels: hand-written sm_90a kernels or the torch/cuDNN library reference")
  add("--seed", type=int, default=0, help="Seed of the parameter initialisation and of the input streams")
  add("--dtype", type=str, default="auto", choices=("auto", "bf16", "tf32", "fp32"), help="Compute precision on the GPU: bf16 tensor-core products (default), or fp32 storage with TF32 products (the precision class of the fp32 reference); fp32 on CPU")
  add("--debug-checksum", action="store_true", default=False, help="Check after every step that all ranks hold bit-identical parameters")
  add("--authenticate", action="store_true", default=False, help="Sign every published gradient (ed25519) and verify before aggregating; slices failing the check become NaN")
  add("--worker-momentum", type=float, default=0.0, help="Worker momentum beta in [0, 1): every worker submits its momentum m <- beta m + (1 - dampening) g instead of its gradient (0 with a zero dampening: off)")
  add("--worker-momentum-dampening", type=float, default=0.0, help="Dampening of the worker momentum in [0, 1)")
  return parser


def _init_distributed(use_gpu):
  """Join the torchrun world if any. Returns (rank, world, local rank, device)."""
  world = int(os.environ.get("WORLD_SIZE", "1"))
  rank = int(os.environ.get("RANK", "0"))
  local = int(os.environ.get("LOCAL_RANK", "0"))
  cuda = use_gpu and torch.cuda.is_available()
  device = torch.device("cuda", local % max(1, torch.cuda.device_count())) if cuda else torch.device("cpu")
  if cuda:
    torch.cuda.set_device(device)
  if world > 1 and not dist.is_initialized():
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29500")
    if cuda:
      dist.init_process_group("nccl", rank=rank, world_size=world, device_id=device)
    else:
      dist.init_process_group("gloo", rank=rank, world_size=world)
  return rank, world, local, device



# ---------------------------------------------------------------------------- #
# Argument post-processing (same user-visible rules and messages as the reference's `runner.py:233-297`, table-driven here)

def _tee_streams(args):
  """`--stdout-to/--stderr-to FILE`: duplicate (not redirect) the stream into FILE, colours stripped."""
  for attr, stream_name, label in (("stdout_to", "stdout", "standard output"), ("stderr_to", "stderr", "standard error output")):
    target = getattr(args, attr)
    if target == "-":
      continue
    path = pathlib.Path(target)
    tee = tools.MethodCallReplicator(getattr(sys, stream_name), tools.ContextIOWrapper(path.open("w"), nocolor=True))
    setattr(sys, stream_name, tee)
    tee.write("Duplicating " + label + " to " + repr(str(path.resolve())) + os.linesep)


def _validate(args):
  """Fatal problems raise `UserException`, suspicious settings only warn; list arguments left out become empty lists."""
  n, f, real = args.nb_workers, args.nb_decl_byz_workers, args.nb_real_byz_workers
  if bool(args.client) == bool(args.server):
    raise tools.UserException("One and only one of '--client' and '--server' must be specified")
  if args.server:
    args.server = tools.cluster_parse(args.server)
    missing = [job for job in (args.ps_job_name, args.wk_job_name, args.ev_job_name) if job not in args.server]
    if missing:
      raise tools.UserException("Given cluster specification does not include a " + repr(missing[0]) + " job")
  fatal = (
    (n <= 0, "Expected at least one non-Byzantine worker"),
    (n < real, "Got more real Byzantine workers (" + repr(real) + ") than total number of workers (" + repr(n) + ")"))
  for failed, message in fatal:
    if failed:
      raise tools.UserException(message)
  advisories = (
    (n <= 2 * f, "Got more declared Byzantine workers (" + repr(f) + ") than half the total number of workers (" + repr(n) + ")"),
    (f < real, "Got more real Byzantine workers (" + repr(real) + ") than declared number of Byzantine workers (" + repr(f) + ")"),
    (args.use_tpu or args.reuse_tpu, "There is no TPU on an H100 box: '--use-tpu/--reuse-tpu' are accepted and ignored"),
    (args.MPI, "'--MPI' is accepted for compatibility: ranks communicate through peer-mapped memory (NVLink) and NCCL/gloo"))
  for suspicious, message in advisories:
    if suspicious:
      tools.warning(message)
  for name in ("experiment_args", "aggregator_args", "learning_rate_args", "optimizer_args", "attack_args"):
    if getattr(args, name) is None:
      setattr(args, name, [])


def _resolve_outputs(args):
  """Evaluation file and summary directory default into the checkpoint directory; "-" switches either off."""
  def resolve(value, default):
    if value == "-":
      return ""
    return value if value else default
  base = args.checkpoint_dir
  args.evaluation_file = resolve(args.evaluation_file, str(pathlib.PurePath(base) / config.default_evaluation_file_name) if base else "")
  args.summary_dir = resolve(args.summary_dir, base if base else "")


def _device_preferences(args):
  """(preference order of device types, types that may host several entities): TPU > GPU > CPU; `--reuse-X` implies `--use-X`."""
  args.use_gpu = args.use_gpu or args.reuse_gpu
  args.use_tpu = args.use_tpu or args.reuse_tpu
  wanted = [("TPU", args.use_tpu, args.reuse_tpu), ("GPU", args.use_gpu, args.reuse_gpu), ("CPU", True, True)]
  return tuple(kind for kind, use, _ in wanted if use), tuple(kind for kind, _, reuse in wanted if reuse)


def main(argv=None):
  global exit_pending
  exit_pending = False
  tools.install()
  tools.success("Python module loading phase...")
  if os.environ.get("AGB_PRINT_ROOT"):
    print("package root: " + str(pathlib.Path(__file__).resolve().parents[2]))
  if threading.current_thread() is threading.main_thread():
    signal.signal(signal.SIGINT, mark_exit)
    signal.signal(signal.SIGTERM, mark_exit)

  # -------------------------------------------------------------------------- #
  tools.success("Command line parsing phase...")
  parser = make_parser()
  with tools.Context("args", "info"):
    args = parser.parse_args(sys.argv[1:] if argv is None else argv)
    _tee_streams(args)
    _validate(args)
    _resolve_outputs(args)
    nb_nonbyz_workers = args.nb_workers - args.nb_real_byz_workers
    device_prefs, device_reuse = _device_preferences(args)
    rank, world, local, device = _init_distributed(args.use_gpu)
    if rank != 0:
      tools.set_rank_tag("r" + str(rank))
    quiet = rank != 0
    if not quiet:
      print("Using a total of " + repr(args.nb_workers) + " worker(s):")
      print("· " + repr(nb_nonbyz_workers) + " non-Byzantine worker(s)")
      print("· " + repr(args.nb_decl_byz_workers) + " declared Byzantine worker(s)")
      print("  " + repr(args.nb_real_byz_workers) + " real Byzantine worker(s)")
      tools.print_args("experiment", args.experiment, args.experiment_args, head="")
      tools.print_args("gradient aggregation rule", args.aggregator, args.aggregator_args, head="")
      tools.print_args("learning rate", args.learning_rate, args.learning_rate_args, head="")
      tools.print_args("optimizer", args.optimizer, args.optimizer_args, head="")
      tools.print_args("attack", args.attack, args.attack_args, head="")
  if exit_pending:
    return 0

  # -------------------------------------------------------------------------- #
  if not quiet:
    tools.success("Cluster analysis and allocation phase...")
  with tools.Context("cluster", "info"):
    if args.server and not quiet:
      tools.info("Acting as node " + args.ps_job_name + ":0 in the cluster (" + str(world) + " rank(s), device " + str(device) + ")")
    gpus = [(r % max(1, torch.cuda.device_count())) if device.type == "cuda" else None for r in range(world)]
    cluster_mgr = cluster.Manager.from_world(world, gpus, args.server if args.server else None, args.ps_job_name, args.wk_job_name, args.ev_job_name, devs=device_prefs, reuse=device_reuse)
    attacked = bool(args.attack) and args.nb_real_byz_workers > 0
    nb_instantiated = args.nb_workers if attacked else nb_nonbyz_workers
    wk_devices = cluster_mgr.allocate("worker", nb_instantiated, jobs={args.wk_job_name})
    if wk_devices is None:
      raise tools.UserException("Unable to allocate " + repr(nb_instantiated) + " devices for the workers on the cluster" + ("" if args.reuse_gpu or device.type != "cuda" else " (several workers per GPU need '--reuse-gpu')"))
    ps_device = cluster_mgr.allocate("ps", 1, jobs={args.ps_job_name})
    if ps_device is None:
      raise tools.UserException("Unable to allocate a device for the parameter server on the cluster")
    ev_device = cluster_mgr.allocate("eval", 1, jobs={args.ev_job_name})
    if ev_device is None:
      raise tools.UserException("Unable to allocate a device for the evaluator on the cluster")
    if not quiet:
      cluster_mgr.report()
    if nb_instantiated % world != 0:
      raise tools.UserException("The %d instantiated workers cannot be spread evenly over %d rank(s)" % (nb_instantiated, world))
    per_rank = {}
    placement = []
    for job, task, devtype, devid in wk_devices:
      task = int(task)
      placement.append((task, per_rank.get(task, 0)))
      per_rank[task] = per_rank.get(task, 0) + 1
    if len(set(per_rank.values())) > 1 or len(per_rank) != world:
      placement = None  # fall back to the contiguous layout
  if exit_pending:
    return 0

  # -------------------------------------------------------------------------- #
  if not quiet:
    tools.success("Graph construction phase...")
  with tools.Context("graph", "info"):
    experiment = experiments.instantiate(args.experiment, args.experiment_args)
    aggregator = aggregators.instantiate(args.aggregator, args.nb_workers, args.nb_decl_byz_workers, args.aggregator_args)
    attack = attacks.instantiate(args.attack, args.nb_workers, args.nb_real_byz_workers, args.attack_args) if attacked else None
    engine = args.engine
    if nb_instantiated != args.nb_workers and engine in ("auto", "fused"):
      engine = "baseline" if device.type == "cuda" else "host"  # absent workers: the GAR sees fewer rows than declared (reference behaviour)
    graph_mgr = Manager(experiment, aggregator, nb_instantiated, args.optimizer, args.optimizer_args, args.learning_rate, args.learning_rate_args,
                        (args.l1_regularize, args.l2_regularize), trace=args.trace, attack=attack, nb_real_byz=args.nb_real_byz_workers if attacked else 0,
                        device=device, engine=engine, backend=args.nn_backend, seed=args.seed, placement=placement, debug_checksum=args.debug_checksum, authenticate=args.authenticate,
                        worker_momentum=args.worker_momentum, worker_momentum_dampening=args.worker_momentum_dampening,
                        dtype={"bf16": torch.bfloat16, "tf32": torch.float32, "fp32": torch.float32}.get(args.dtype))
  if exit_pending:
    return 0

  # -------------------------------------------------------------------------- #
  if not quiet:
    tools.success("Training and evaluation session phase...")
  lock = threading.RLock()
  stop_event = threading.Event()
  threads = []
  inline = []  # (flag, service, cadence) for the multi-rank inline driver
  total_runtime = first_runtime = -1.
  graph_runtime = 0.
  rawstep = 0
  try:
    with tools.Context("checkpoint", "info"):
      restored = False
      checkpoints = None
      if args.checkpoint_dir:
        checkpoints = tools.Checkpoints(args.checkpoint_dir)
        if checkpoints.can_restore():
          if not quiet:
            print("Loading latest checkpoint in " + repr(args.checkpoint_dir) + "...")
          graph_mgr.load_state_dict(checkpoints.restore())
          restored = True
        elif not quiet:
          print("No checkpoint to restore")
      if exit_pending:
        raise KeyboardInterrupt
    if not quiet:
      tools.success("Launching evaluation, checkpoint and summary threads...")
    evaluator = services.Evaluator(graph_mgr, args.evaluation_file if rank == 0 else "")
    eval_cadence = services.Cadence(args.evaluation_delta, args.evaluation_period)
    meta = {"argv": sys.argv if argv is None else list(argv), "experiment": args.experiment, "aggregator": args.aggregator, "nb_workers": args.nb_workers}
    ckpt_service = services.Checkpointer(graph_mgr, checkpoints, meta, write=rank == 0) if checkpoints is not None else None
    ckpt_cadence = services.Cadence(args.checkpoint_delta, args.checkpoint_period, restored, graph_mgr.step)
    sum_service = services.Summarizer(graph_mgr, evaluator, args.summary_dir) if (args.summary_dir and rank == 0) else None
    sum_cadence = services.Cadence(args.summary_delta, args.summary_period, restored, graph_mgr.step)
    if world == 1:
      first_eval = threading.Event()
      threads.append(services.ServiceThread("test", evaluator, eval_cadence, graph_mgr, lock, stop_event, first_eval))
      if ckpt_service is not None:
        threads.append(services.ServiceThread("checkpoint", ckpt_service, ckpt_cadence, graph_mgr, lock, stop_event))
      if sum_service is not None:
        threads.append(services.ServiceThread("summary", sum_service, sum_cadence, graph_mgr, lock, stop_event))
      for thread in threads:
        thread.start()
      first_eval.wait()
    else:
      inline = [(services.FLAG_EVAL, evaluator, eval_cadence)]
      if ckpt_service is not None:
        inline.append((services.FLAG_CHECKPOINT, ckpt_service, ckpt_cadence))
      if sum_service is not None or rank != 0:
        inline.append((services.FLAG_SUMMARY, sum_service, sum_cadence))
    if exit_pending:
      raise KeyboardInterrupt

    def run_inline(final=False):
      """Rank 0 decides which services are due; every rank executes the collective ones."""
      flags = torch.zeros(1, dtype=torch.int64, device=device)
      if rank == 0:
        now, value = time.time(), 0
        for flag, service, cadence in inline:
          if not cadence.disabled and (final or cadence.due(graph_mgr.step, now)):
            value |= flag
        if exit_pending:
          value |= services.FLAG_STOP
        flags[0] = value
      dist.broadcast(flags, src=0)
      value = int(flags.item())
      for flag, service, cadence in inline:
        if value & flag:
          if flag == services.FLAG_EVAL and rank != 0:
            continue  # evaluation is local to rank 0
          if service is not None:
            service.run(graph_mgr.step)
          cadence.mark(graph_mgr.step)
      if value & (services.FLAG_EVAL | services.FLAG_CHECKPOINT | services.FLAG_SUMMARY):
        # rank 0 just spent an arbitrary time evaluating / writing files: re-align the ranks on the host before anyone launches
        # the next step's aggregation kernel (whose entry barrier spins on every peer's flag)
        dist.barrier()
      return bool(value & services.FLAG_STOP)

    if world > 1:
      run_inline()
    if not quiet:
      tools.success("Actual training...")
    offstep = graph_mgr.step
    total_runtime = time.time()
    poll_every = 1
    while args.max_step <= 0 or rawstep < args.max_step:
      step = rawstep + offstep
      runtime_begin = time.time()
      with lock:
        res = float(graph_mgr.train())  # one training step; the float() is the device->host read of the loss
      if first_runtime < 0.:
        first_runtime = time.time() - runtime_begin
      else:
        graph_runtime += time.time() - runtime_begin
      rawstep += 1
      if math.isfinite(res):
        if not quiet:
          tools.info("Step " + str(step) + ": total loss = " + str(res), context="train")
      else:
        if not quiet:
          tools.info("Step " + str(step) + ": total loss = NaN", context="train")
        raise tools.UserException("Model diverged with loss = NaN")
      for thread in threads:
        if thread.error is not None:
          raise thread.error
      if world > 1 and rawstep % poll_every == 0:
        if run_inline():
          break
      elif exit_pending:
        break
  except KeyboardInterrupt:
    pass
  finally:
    if total_runtime > 0.:
      total_runtime = time.time() - total_runtime
    stop_event.set()
    for thread in threads:
      thread.join()
    if world > 1 and inline and dist.is_initialized() and sys.exc_info()[0] is None:
      run_inline(final=True)
    for _, service, _ in inline:
      if service is not None:
        service.close()
    graph_mgr.close()
    if total_runtime > 0. and not quiet:
      offgraph_runtime = total_runtime - graph_runtime - max(first_runtime, 0.)
      text = " In-graph:   " + str(graph_runtime) + " s (" + str(graph_runtime / total_runtime * 100.) + " %)" + os.linesep
      if first_runtime > 0.:
        text += "           + " + str(first_runtime) + " s (" + str(first_runtime / total_runtime * 100.) + " %)" + os.linesep
      text += " Off-graph:  " + str(offgraph_runtime) + " s (" + str(offgraph_runtime / total_runtime * 100.) + " %)" + os.linesep
      text += " Throughput: " + str(rawstep / total_runtime) + " step(s)/s (all steps)" + os.linesep
      if first_runtime > 0. and total_runtime > first_runtime:
        text += "             " + str(max(rawstep - 1, 0) / (total_runtime - first_runtime)) + " step(s)/s (excluding 1st step)"
      tools.info(text, context="perf")
      phases = graph_mgr.tracer.report()
      if args.trace and phases:
        for what, entry in phases.items():
          tools.trace(" %s: %d call(s), host %.3f s, device %s ms" % (what, entry["count"], entry["host_s"], "n/a" if entry["device_ms"] is None else "%.3f" % entry["device_ms"]), context="perf")

  if args.server and not args.no_wait and rank == 0 and threading.current_thread() is threading.main_thread():
    try:
      with tools.Context(None, "success"):
        sys.stdout.write("Current process is acting as a cluster node: waiting for any signal...")
        sys.stdout.flush()
      signal.pause()
    except KeyboardInterrupt:
      pass
    finally:
      print("")
  if dist.is_initialized():
    dist.destroy_process_group()
  return 0


if __name__ == "__main__":
  sys.exit(main())

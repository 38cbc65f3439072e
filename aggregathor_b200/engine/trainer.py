"""Training step builder (reference: `graph.Manager`, `graph.py:204-315`).

The reference assembles one TF graph: per-worker loss/gradient subgraphs pinned to the workers' devices, the GAR
and `apply_gradients` pinned to the PS, an evaluator replica, and `train_tn = total_loss` gated on the update op.
`Manager` keeps that surface (`step`, `rate`, `optimizer`, `total_loss`, `train()`≈`sess.run(train_tn)`,
`evaluate()`≈`sess.run(eval_tns)`) on an SPMD runtime: every rank hosts `w = n / R` logical workers and owns 1/R
of the parameter server (see `parallel/aggregation.py`).

One synchronous step on a rank:
  1. for each local worker: next batch (already prefetched to the device), forward, loss, backward — gradients are
     written by the layer kernels directly into that worker's row of the peer-mapped `[w, d]` gradient matrix;
  2. optional l1 / l2 regularisation gradient (same formulas as `graph.py:125-139`);
  2b. optional worker momentum (`worker_momentum` beta, `worker_momentum_dampening` delta; El Mhamdi et al., "Distributed Momentum for
     Byzantine-resilient SGD"): every local row becomes its worker's momentum M <- beta M + (1 - delta) G, before anything else
     reads it — a real Byzantine worker keeps its honest momentum, the attack then transforms or replaces what is submitted;
  3. real Byzantine workers overwrite their row with the selected attack (omniscient attacks: the aggregation engine crafts the
     Byzantine rows from the honest ones, a collective call on every rank; data poisoning: nothing, step 1 already trained the
     Byzantine workers on flipped labels through `Context.flip_from`, or on triggered and relabelled samples with scaled loss
     gradients through `Context.backdoor`);
  4. the aggregation engine runs (fused kernel: gather + GAR + optimizer + parameter broadcast), after the optional pre-aggregation
     (`pre_aggregation="nnm"`: nearest-neighbour mixing of the gathered rows, Allouah et al., "Fixing by Mixing"; "arc": adaptive
     robust clipping, Allouah et al., "Boosting Robustness by Clipping Gradients in Distributed Learning"; "arc+nnm": both;
     "bucketing": means of shuffled buckets of s rows, Karimireddy, He & Jaggi, "Byzantine-Robust Learning on Heterogeneous Datasets
     via Bucketing");
  5. the bf16 compute copy of the parameters is refreshed (unless the fused kernel already wrote it).
With a rule that needs a trusted root gradient (`fltrust`), rank 0 alone also runs, in step 1, one unbatched forward/backward on a
batch of the experiment's root dataset into the engine's root row (never flipped, never poisoned, its loss not reported): the ranks run
in lock-step, so one root pass costs the same wall time as one on every rank, and one root row owned by rank 0 gives every engine the
same root gradient at any rank count.
"""

import os
import time

import torch
import torch.distributed as dist

from .. import tools
from ..models import Context
from ..ops import gar as gar_ops
from ..parallel.aggregation import make_aggregation
from .flat import FlatLayout, regularization
from .optimizers import optimizers
from .schedules import build, learning_rates


def _default_device():
  if torch.cuda.is_available():
    return torch.device("cuda", torch.cuda.current_device())
  return torch.device("cpu")


class Manager:
  """Full training + evaluation state of one rank."""

  def __init__(self, experiment, aggregator, nbworkers, optimizer="sgd", optimizer_args=None, learning_rate="fixed", learning_rate_args=None,
               regularizations=(-1., -1.), trace=False, *, attack=None, nb_real_byz=0, device=None, group=None, engine="auto", backend="auto",
               dtype=None, seed=0, placement=None, debug_checksum=False, engine_args=None, use_graphs=None, authenticate=False,
               worker_momentum=0.0, worker_momentum_dampening=0.0, pre_aggregation="none", nb_decl_byz=None, bucket_size=None, bucketing_seed=0):
    """`pre_aggregation`: "none", "nnm" (every row replaced by the mean of its n - f nearest rows before the rule), "arc" (adaptive
    robust clipping: the floor(2 f (n - f) / n) rows of largest norm clipped to the norm of the largest row left alone) or "arc+nnm"
    (ARC, then NNM), with f = `nb_decl_byz`, the declared Byzantine workers (default: the rule's own f); or "bucketing" (the rows,
    shuffled by a permutation keyed by `bucketing_seed` and the update number, replaced by the means of buckets of `bucket_size` rows;
    `aggregator` is then built for ceil(nbworkers / bucket_size) workers)."""
    from ..aggregators import _ops
    self.pre_aggregation = _ops.check_pre_aggregation(pre_aggregation, bucket_size)   # None, "nnm", "arc", "arc+nnm" or "bucketing"
    # (beta, c = 1 - dampening) in fp32; beta = dampening = 0 is off: no buffer, no kernel, the step is unchanged
    self.momentum = _ops.check_worker_momentum(worker_momentum, worker_momentum_dampening)
    self.momentum_on = self.momentum[0] != 0.0 or _ops.fp32(worker_momentum_dampening) != 0.0
    self.needs_root = bool(getattr(aggregator, "needs_root", False))
    if self.needs_root and self.momentum_on:
      raise tools.UserException("%s compares every row with a raw root gradient: it cannot be combined with --worker-momentum" % type(aggregator).__name__)
    if authenticate and getattr(attack, "omniscient", False):
      raise tools.UserException("Omniscient attacks craft the Byzantine rows on every rank: they cannot be combined with '--authenticate'")
    self.device = torch.device(device) if device is not None else _default_device()
    if self.device.type == "cuda" and self.device.index is None:
      self.device = torch.device("cuda", torch.cuda.current_device())
    self.group = group
    self.rank = dist.get_rank(group) if dist.is_initialized() else 0
    self.world = dist.get_world_size(group) if dist.is_initialized() else 1
    self.experiment, self.aggregator, self.n = experiment, aggregator, nbworkers
    self.l1, self.l2 = regularizations
    self.tracer = tools.Tracer(enabled=trace, cuda=self.device.type == "cuda")
    self.debug_checksum = debug_checksum
    cuda = self.device.type == "cuda"
    self.dtype = dtype if dtype is not None else (torch.bfloat16 if cuda else torch.float32)
    if backend == "auto":
      backend = "native" if cuda else "torch"
    self.backend = backend
    # -- learning rate, optimizer ------------------------------------------------- #
    self.rate = build(learning_rates, "learning rate decay", learning_rate, learning_rate_args)
    self.optimizer = build(optimizers, "optimizer", optimizer, optimizer_args)
    # -- model, layout -------------------------------------------------------------- #
    self.model = experiment.model()
    self.layout = FlatLayout()
    state_shapes = {}
    self.model.declare(self.layout, state_shapes)
    self.layout.freeze()
    # -- aggregation engine (owns params + gradient rows) -------------------------- #
    engine_args = dict(engine_args or {})
    self._bucket_layers = {}
    # phase A reads the rows during the backward pass: nothing may rewrite them afterwards (attacks, signing, worker momentum); with
    # a pre-aggregation the rule's distances are those of the mixed or clipped rows, which exist only once every row is complete.
    # Data poisoning rewrites no row: its Byzantine rows are complete when the backward pass ends, like the honest ones.
    self._rewrites_rows = attack is not None and not getattr(attack, "poisons_data", False)
    plain_step = (not self._rewrites_rows and not authenticate and not ((self.l1 or -1.) > 0. or (self.l2 or -1.) > 0.) and not self.momentum_on
                  and self.pre_aggregation is None)
    if cuda and engine in ("auto", "fused") and aggregator.fused_spec() is not None:
      engine_args.setdefault("device_state", True)
      # The bucketed distance pass moves the gather + distance work of Krum / Bulyan under the backward pass (`gar_phase_a_kernel` on a side
      # stream, bucket by bucket). The step is bandwidth- and launch-bound rather than waiting on NVLink, and the finish kernel alone
      # is not shorter than the single-launch aggregation (flag barriers and the parameter broadcast dominate, not the gather), so the
      # pass is opt-in: AGB_OVERLAP=1 for single-worker ranks of multi-rank jobs, =2 always.
      overlap = os.environ.get("AGB_OVERLAP", "0")
      single_worker_ranks = self.world > 1 and nbworkers == self.world
      if plain_step and aggregator.fused_spec().rule in ("krum", "bulyan", "mda", "smea") and (overlap == "2" or (overlap not in ("", "0") and single_worker_ranks)) and "buckets" not in engine_args:
        buckets, self._bucket_layers = self._plan_buckets()
        if len(buckets) > 1:
          engine_args["buckets"] = buckets
    mix = dict(pre_aggregation=self.pre_aggregation, nb_decl_byz=nb_decl_byz)
    if self.pre_aggregation == "bucketing":
      mix.update(bucket_size=bucket_size, bucketing_seed=bucketing_seed)
    try:
      self.aggregation = make_aggregation(engine, aggregator, self.layout, nbworkers, self.optimizer, group, self.device, **mix, **engine_args)
    except TypeError:   # engines without these options (host, baseline)
      self.aggregation = make_aggregation(engine, aggregator, self.layout, nbworkers, self.optimizer, group, self.device, **mix)
    if not getattr(self.aggregation, "overlappable", False):
      self._bucket_layers = {}
    self._side_stream = None
    if cuda and backend == "native" and self.aggregation.w == 1 and "AGB_PDL" not in os.environ and "AGB_WGRAD_STREAM" not in os.environ and os.environ.get("AGB_LAUNCH_OVERLAP", "1") != "0":
      from ..ops import nn_native
      nn_native.set_launch_overlap(True)   # one batch-32 worker per rank: small kernels, overlap their launches and the weight gradients
    self.w = self.aggregation.w
    self.params = self.aggregation.params
    self.grads = self.aggregation.grads
    # worker momentum: one fp32 row per local row of `grads` (same local index), +0 at the start
    self.worker_momentum = torch.zeros((self.w, self.layout.padded_size), dtype=torch.float32, device=self.device) if self.momentum_on else None
    self.states = {name: torch.zeros(shape, dtype=torch.float32, device=self.device) for name, shape in state_shapes.items()}
    # identical initial parameters on every rank: same seed, CPU generator, then copy
    generator = torch.Generator().manual_seed(seed)
    init = torch.zeros(self.layout.padded_size, dtype=torch.float32)
    init_states = {name: torch.zeros(shape, dtype=torch.float32) for name, shape in state_shapes.items()}
    self.model.initialize(self.layout.views(init), init_states, generator)
    self.params.copy_(init)
    for name, value in init_states.items():
      self.states[name].copy_(value)
    self.master_views = self.layout.views(self.params)
    if self.dtype != torch.float32:
      fused_copy = getattr(self.aggregation, "params_bf16", None)
      self._weights_flat = fused_copy if fused_copy is not None else torch.zeros(self.layout.padded_size, dtype=self.dtype, device=self.device)
      self._weights_by_kernel = fused_copy is not None
      self.weight_views = self.layout.views(self._weights_flat)
    else:
      self._weights_flat, self._weights_by_kernel, self.weight_views = None, True, self.master_views
    self._refresh_weights(force=True)
    # -- workers -------------------------------------------------------------------- #
    if placement is None:
      placement = [(i // self.w, i % self.w) for i in range(nbworkers)]
    self.placement = placement
    self.local_workers = [i for i, (rank, _) in enumerate(placement) if rank == self.rank]
    self.contexts = []
    self._dropout_gen = torch.Generator(device=self.device).manual_seed(seed * 977 + self.rank + 1)
    for i in self.local_workers:
      ctx = Context(self.backend, True, self.dtype, self.device)
      ctx.weights, ctx.master, ctx.state = self.weight_views, self.master_views, self.states
      ctx.grads = self.layout.views(self.grads[placement[i][1]])
      ctx.generator = self._dropout_gen
      ctx.worker_id, ctx.nbworkers = i, nbworkers
      self.contexts.append(ctx)
    # all local workers in one pass (per-worker BN statistics / losses / gradients): needs rows 0..w-1 in worker order
    base = type(experiment).__mro__[-2]
    contiguous_rows = [placement[i][1] for i in self.local_workers] == list(range(len(self.local_workers)))
    want_batched = os.environ.get("AGB_BATCH_WORKERS", "1") != "0"
    self.batched = (want_batched and cuda and len(self.local_workers) > 1 and contiguous_rows and not self._has_dropout(self.model.root)
                    and type(experiment).losses is base.losses and type(experiment).losses_batched is base.losses_batched)
    self.batched_ctx = None
    if self.batched:
      bctx = Context(self.backend, True, self.dtype, self.device)
      bctx.weights, bctx.master, bctx.state = self.weight_views, self.master_views, self.states
      bctx.grads = self.layout.views(self.grads[0])
      bctx.generator = self._dropout_gen
      bctx.groups, bctx.group_stride = len(self.local_workers), self.grads.stride(0)
      bctx.worker_id, bctx.nbworkers = self.local_workers[0], nbworkers
      self.batched_ctx = bctx
    self.eval_ctx = Context(self.backend, False, self.dtype, self.device)
    self.eval_ctx.weights, self.eval_ctx.master, self.eval_ctx.state = self.weight_views, self.master_views, self.states
    self.eval_ctx.generator = self._dropout_gen
    self.streams = [experiment.train_stream(i, nbworkers, self.device) for i in self.local_workers]
    # FLTrust: the root pass of rank 0, with its own training context whose gradients are the engine's root row, and its own copy of
    # the model state (batch-norm moving averages), so that every rank keeps the same state
    self.root_ctx = self.root_stream = None
    if self.needs_root:
      experiment.root_indices(aggregator.root_size)   # the same checks on every rank
      if self.rank == 0:
        ctx = Context(self.backend, True, self.dtype, self.device)
        ctx.weights, ctx.master = self.weight_views, self.master_views
        ctx.state = {name: value.clone() for name, value in self.states.items()}
        ctx.grads = self.layout.views(self.aggregation.root)
        ctx.generator = self._dropout_gen
        ctx.worker_id, ctx.nbworkers = nbworkers, nbworkers   # one past the workers: its own augmentation stream
        ctx.flip_from = ctx.backdoor = None
        self.root_ctx = ctx
        self.root_stream = experiment.root_stream(aggregator.root_size, self.device)
    self._stream_group = None
    if cuda and os.environ.get("AGB_GROUP_STREAMS", "1") not in ("", "0"):
      from ..experiments._data import StreamGroup
      if StreamGroup.eligible(self.streams):
        self._stream_group = StreamGroup(self.streams)   # one pinned slab + one H2D copy per step for all the workers of this rank
        self._grouped_source = self.streams              # (only while `self.streams` is still this very list: callers may swap it)
    # -- attack --------------------------------------------------------------------- #
    self.nb_real_byz = nb_real_byz
    self.attack = attack
    self.byzantine = set(range(nbworkers - nb_real_byz, nbworkers)) if (attack is not None and nb_real_byz > 0) else set()
    self._attack_state = {i: {} for i in self.byzantine}
    if self.byzantine and getattr(attack, "mode", None) == "mimic":   # created now, so that a restored checkpoint finds it
      self.aggregation.mimic_state()
    # the backdoor: its evaluation set and the context that stamps the trigger on all of it, checked on every rank
    self.backdoor_ctx = self._backdoor_batch = None
    if self.byzantine and getattr(attack, "poisons_data", False) and not attack.flips_labels:
      attack.check_target(experiment.num_classes)
      q = attack.poisoned_rows(int(experiment.args["batch-size"]))
      self._backdoor_batch = experiment.backdoor_batch(attack.target)
      ctx = Context(self.backend, False, self.dtype, self.device)
      ctx.weights, ctx.master, ctx.state = self.weight_views, self.master_views, self.states
      ctx.generator = self._dropout_gen
      ctx.backdoor = (0, len(self._backdoor_batch[1]), attack.target, 1.0)
      self.backdoor_ctx = ctx
    if self.byzantine and getattr(attack, "poisons_data", False):   # training contexts only: `eval_ctx` is never poisoned
      def poison(ctx, first):   # the groups >= first of the context's batch are poisoned (None: none)
        if attack.flips_labels:
          ctx.flip_from = first
        else:
          ctx.backdoor = None if first is None else (first, q, attack.target, attack.scale)
      for ctx, i in zip(self.contexts, self.local_workers):
        poison(ctx, 0 if i in self.byzantine else None)
      if self.batched_ctx is not None:
        # group j of the batched pass is local worker j (ascending ids, rows 0..w-1): the Byzantine workers, the last k ids, are
        # the groups from the number of honest local workers on
        honest = sum(i not in self.byzantine for i in self.local_workers)
        assert self.local_workers == sorted(self.local_workers) and all((i in self.byzantine) == (j >= honest) for j, i in enumerate(self.local_workers))
        poison(self.batched_ctx, honest if honest < len(self.local_workers) else None)
    # rows in the gathered matrix (slots) of the Byzantine workers, as the aggregation engines address them
    self.byzantine_slots = sorted(placement[i][0] * self.w + placement[i][1] for i in self.byzantine)
    # -- gradient authentication (opt-in; reference: signed worker -> PS messages of the hardened transport) -- #
    self.authenticator = None
    if authenticate:
      from ..parallel.signing import Authenticator
      self.authenticator = Authenticator(self.layout, nbworkers, group)
    # -- counters ------------------------------------------------------------------- #
    self.step = 0
    self.total_loss = None
    self._loss_buf = torch.zeros(1, dtype=torch.float32, device=self.device)
    self.h2d_bytes_per_step = sum(getattr(s, "h2d_bytes", 0) for s in self.streams)
    # -- CUDA graph of the workers' forward/backward ---------------------------------- #
    if use_graphs is None:
      use_graphs = (cuda and not os.environ.get("AGB_NO_GRAPH") and not self._has_dropout(self.model.root) and not getattr(experiment, "stochastic_preprocess", False)
                    and type(experiment).losses is type(experiment).__mro__[-2].losses)
    self.use_graphs = bool(use_graphs) and cuda
    self._graph = None
    self._graph_whole = False
    self._overlap_armed = False  # set for the duration of a step once `aggregation.prepare()` has run (phase A needs the step's scalars)
    self._graph_warmup = 2       # eager steps before capture (lazy kernel attributes, workspaces, autotuning)
    self._graph_launches = 0
    tools.info("Model %r: %d variables, d = %d (padded %d); %d worker(s) on this rank%s; compute dtype %s; nn backend %r; engine %r" % (
      self.model.name, len(self.layout.names), self.layout.size, self.layout.padded_size, len(self.local_workers), " (batched in one pass)" if self.batched else "",
      str(self.dtype).replace("torch.", ""), self.backend, self.aggregation.name), context="graph")

  # ---------------------------------------------------------------------------- #
  def _refresh_weights(self, force=False):
    if self._weights_flat is None:
      return
    if self._weights_by_kernel and not force:
      return
    if self.device.type == "cuda" and self.dtype == torch.bfloat16:
      gar_ops.cast_bf16_(self.params, self._weights_flat)
    else:
      self._weights_flat.copy_(self.params)

  @staticmethod
  def _has_dropout(module):
    from ..models.core import DropPath, Dropout
    if isinstance(module, (Dropout, DropPath)) and module.keep_prob < 1.0:
      return True
    return any(Manager._has_dropout(child) for child in module.children())

  @property
  def _whole_step_graph(self):
    """The captured graph holds the aggregation too (fused engine with device-resident step state, nothing host-driven in between)."""
    return (getattr(self.aggregation, "device_state", False) and not self._rewrites_rows and self.authenticator is None
            and not ((self.l1 or -1.) > 0. or (self.l2 or -1.) > 0.) and os.environ.get("AGB_GRAPH_AGGREGATION", "1") not in ("", "0"))

  def _capture(self, batches, root_batch=None):
    """Record every local worker's forward + backward — and, with the fused engine, the aggregation kernels and the refresh of the
    compute copy of the parameters — into one CUDA graph (static shapes, static buffers)."""
    from ..ops import counters
    uniform = len(batches) > 1 and all(x.shape == batches[0][0].shape and x.dtype == batches[0][0].dtype and y.shape == batches[0][1].shape and y.dtype == batches[0][1].dtype
                                       for x, y in batches)
    if uniform:   # static inputs as two slabs (views per worker): a grouped input stream refreshes them with one copy each
      slab_x, slab_y = torch.stack([x for x, _ in batches]), torch.stack([y for _, y in batches])
      self._static_batches, self._static_slabs = [(slab_x[j], slab_y[j]) for j in range(len(batches))], (slab_x, slab_y)
    else:
      self._static_batches, self._static_slabs = [(x.clone(), y.clone()) for x, y in batches], (None, None)
    # FLTrust: the static root batch, refreshed before every replay as the workers' slabs
    self._static_root = (root_batch[0].clone(), root_batch[1].clone()) if root_batch is not None else None
    torch.cuda.synchronize(self.device)
    if self.world > 1:
      dist.barrier(group=self.group)   # capture is slow and its kernels do not run: keep the ranks aligned around it
    graph = torch.cuda.CUDAGraph()
    before = counters.launches
    whole = self._whole_step_graph
    try:
      # thread-local capture: the input pipelines' producer threads keep allocating, copying and synchronising on their own streams
      # while this thread captures. Under the default global mode any such call in another thread fails and invalidates the
      # capture, and a capture that ends that way leaves torch's default CUDA generator in capture mode for the rest of the process.
      with torch.cuda.graph(graph, capture_error_mode="thread_local"):
        self._static_losses = self._run_workers(self._static_batches, None, self._static_root)
        if whole:
          self._apply_momentum()
          self.aggregation.step(stream=None, loss_in=self._static_losses, prepared=True)
          self._refresh_weights()
    except Exception as err:
      tools.warning("CUDA graph capture failed (" + str(err).splitlines()[0] + "): staying in eager mode", context="graph")
      self.use_graphs = False
      torch.cuda.synchronize(self.device)
      return False
    self._graph_launches = counters.launches - before
    self._graph = graph
    self._graph_whole = whole
    tools.info("Captured the workers' forward/backward%s into a CUDA graph (%d native kernel launches per replay)" % (
      " + aggregation" if whole else "", self._graph_launches), context="graph")
    return True

  def _run_workers(self, batches, trace, root_batch=None):
    """Forward + backward of every local worker -> fp32 tensor of per-worker losses; then the root pass on `root_batch` (rank 0 of a
    rule with a root gradient), whose loss is not returned."""
    if self.backend == "native" and self.device.type == "cuda" and not os.environ.get("AGB_NO_PREZERO"):
      # one fill of the whole gradient matrix instead of one per split-K weight gradient; the root row obeys the same contract
      from ..ops import nn_native
      self.grads.zero_()
      if root_batch is not None:
        self.aggregation.root.zero_()
      with nn_native.prezeroed_gradients():
        losses = self._run_workers_inner(batches, trace)
        self._root_pass(root_batch)
        return losses
    losses = self._run_workers_inner(batches, trace)
    self._root_pass(root_batch)
    return losses

  def _root_pass(self, root_batch):
    """One unbatched forward/backward on a root batch into the root row (never poisoned: the model's loss, not the experiment's)."""
    if root_batch is not None:
      inputs, labels = root_batch
      self.model.loss_and_backward(self.experiment.preprocess(inputs, self.root_ctx, True), labels, self.root_ctx)

  def _run_workers_inner(self, batches, trace):
    hooked = self.batched_ctx if (self.batched and trace is None) else (self.contexts[-1] if self.contexts else None)
    overlap = bool(self._bucket_layers) and hooked is not None and self._overlap_armed
    if overlap:   # the bucket of a layer is complete once the LAST local worker has differentiated it
      main = torch.cuda.current_stream(self.device)
      if self._side_stream is None:
        self._side_stream = torch.cuda.Stream(device=self.device, priority=-1)
      side = self._side_stream

      def publish(layer):
        seg = self._bucket_layers.get(id(layer))
        if seg is not None:
          side.wait_stream(main)
          self.aggregation.phase_a(seg, stream=side)
      hooked.backward_hook = publish
    try:
      if self.batched and trace is None:
        losses = self.experiment.losses_batched(self.model, batches, self.batched_ctx).float()
      else:
        per_worker = self.experiment.losses(self.model, batches, self.contexts, trace)
        losses = torch.stack([l.float().reshape(()) for l in per_worker])
    finally:
      if hooked is not None:
        hooked.backward_hook = None
    if overlap:
      main.wait_stream(side)
    return losses

  def _plan_buckets(self):
    """Gradient buckets for the overlapped distance pass: top-level layers in backward order, cut where the accumulated share of the
    parameters passes 50 %, 80 % and 94 % (ResNet-50: logits + block4, block3, block2; the remaining 6 % — the layers whose backward
    finishes last — are handled by the finish kernel itself). Returns ([(lo, hi)] in completion order, {id(layer): bucket})."""
    from ..models.core import Sequential
    root = self.model.root
    if not isinstance(root, Sequential) or len(root.layers) < 4:
      return [], {}
    spans = []
    for layer in root.layers:
      scratch = FlatLayout()
      layer.declare(scratch, {})
      names = scratch.names
      if names:
        lo = min(self.layout.offset(name) for name in names)
        spans.append((layer, lo))
      else:
        spans.append((layer, None))
    total = self.layout.padded_size
    cuts, thresholds, upper, pending = [], [0.5, 0.8, 0.94], total, None
    for layer, lo in reversed(spans):
      if lo is None:
        continue
      share = (total - lo) / total
      if thresholds and share >= thresholds[0] and lo % 4 == 0 and lo < upper and lo > 0:
        cuts.append((layer, lo, upper))
        upper = lo
        while thresholds and share >= thresholds[0]:
          thresholds.pop(0)
    if not cuts:
      return [], {}
    buckets = [(lo, hi) for _, lo, hi in cuts] + [(0, upper)]
    return buckets, {id(layer): index for index, (layer, _, _) in enumerate(cuts)}

  def _replay(self, batches, root_batch=None):
    from ..ops import counters
    if self._static_root is not None:
      self._static_root[0].copy_(root_batch[0], non_blocking=True)
      self._static_root[1].copy_(root_batch[1], non_blocking=True)
    slab_x, slab_y = self._static_slabs
    grouped_x = slab_x is not None and getattr(batches, "x_all", None) is not None and batches.x_all.shape == slab_x.shape
    grouped_y = slab_y is not None and getattr(batches, "y_all", None) is not None and batches.y_all.shape == slab_y.shape
    if grouped_x:
      slab_x.copy_(batches.x_all, non_blocking=True)    # every worker's images in one copy
    if grouped_y:
      slab_y.copy_(batches.y_all, non_blocking=True)
    if not (grouped_x and grouped_y):
      for (sx, sy), (x, y) in zip(self._static_batches, batches):
        if not grouped_x:
          sx.copy_(x, non_blocking=True)
        if not grouped_y:
          sy.copy_(y, non_blocking=True)
    self._graph.replay()
    counters.bump(self._graph_launches)
    return list(self._static_losses.unbind(0))

  def _apply_momentum(self):
    """Worker momentum on every local row (one kernel launch for the rank): M <- beta M + c G, then G <- M."""
    if self.momentum_on:
      gar_ops.worker_momentum_(self.grads, self.worker_momentum, *self.momentum)

  def compute_gradients(self):
    """Phase 1-3 of a step: local workers' losses and gradients (+ regularisation, + attacks). Returns the list of losses."""
    group = self._stream_group
    batches = next(group) if (group is not None and self.streams is self._grouped_source) else [next(stream) for stream in self.streams]
    root_batch = next(self.root_stream) if self.root_stream is not None else None
    trace = self.tracer if self.tracer.enabled else None
    if self.use_graphs and trace is None and self._graph is None and self.step >= self._graph_warmup:
      self._capture(batches, root_batch)
    self._last_step_replayed = self._graph is not None and trace is None
    if self._last_step_replayed:
      losses = self._replay(batches, root_batch)
    else:
      losses = list(self._run_workers(batches, trace, root_batch).unbind(0))
    if (self.l1 is not None and self.l1 > 0.) or (self.l2 is not None and self.l2 > 0.):
      reg_loss, reg_grad = regularization(self.params, self.l1, self.l2)
      for j in range(len(self.local_workers)):
        self.grads[self.placement[self.local_workers[j]][1]].add_(reg_grad)
        losses[j] = losses[j] + reg_loss
      if self.root_ctx is not None:
        self.aggregation.root.add_(reg_grad)
    if not (self._last_step_replayed and self._graph_whole):   # the whole-step graph holds the momentum step
      self._apply_momentum()
    if getattr(self.attack, "omniscient", False):
      if self.byzantine_slots:   # collective: every rank crafts its share, whether or not it hosts a Byzantine worker
        deviation = getattr(self.attack, "deviation", None)   # Min-Max / Min-Sum only: other engines' signatures stay as they were
        extra = {} if deviation is None else {"deviation": deviation}
        if getattr(self.attack, "warmup", None) is not None:   # mimic only
          extra["warmup"] = self.attack.warmup
        for key in ("threshold", "scale", "seed"):   # fang-krum: threshold; fang-trim: scale, seed
          if getattr(self.attack, key, None) is not None:
            extra[key] = getattr(self.attack, key)
        self.aggregation.craft_byzantine(self.byzantine_slots, self.attack.mode, self.attack.coef, **extra)
      return losses
    if not self._rewrites_rows:   # no attack, or data poisoning: the rows are final
      return losses
    forging = self.authenticator is not None and getattr(self.attack, "forges", False)
    for j, i in enumerate(self.local_workers):
      if i in self.byzantine and not forging:
        self.attack.apply(self.grads[self.placement[i][1]], i, self.step, self._attack_state[i])
    return losses

  def authenticate_gradients(self):
    """Sign the local rows, let forging attackers tamper with theirs, exchange the records, verify what this rank will consume."""
    auth = self.authenticator
    # rows are identified by their slot in the gathered matrix (rank * w + local row): the cluster allocation may spread the
    # logical workers over the ranks in any order, the aggregation engines and the records only know slots
    local = [(self.rank * self.w + self.placement[i][1], self.grads[self.placement[i][1]]) for i in self.local_workers]

    def tamper():
      if getattr(self.attack, "forges", False):
        for i in self.local_workers:
          if i in self.byzantine:
            self.attack.apply(self.grads[self.placement[i][1]], i, self.step, self._attack_state[i])

    records = auth.publish(self.step, local, after_sign=tamper)
    return auth.verify(self.step, self.aggregation.visible_rows(), records, self.aggregation.consumed_slices())

  def train(self):
    """One synchronous training step (the reference's `sess.run(train_tn)`); returns the total loss as a 0-d device tensor."""
    rate = self.rate(self.step)
    fused = hasattr(self.aggregation, "prepare")
    if fused:
      self.aggregation.prepare(rate)   # host scalars of the step (stream-ordered, outside any graph)
    self._overlap_armed = fused
    with self.tracer.span("Workers: loss and gradient computation"):
      losses = self.compute_gradients()
    self._overlap_armed = False
    replayed_whole = self._graph is not None and self._graph_whole and self._last_step_replayed
    if not replayed_whole:
      if self.authenticator is not None:
        with self.tracer.span("Authentication: sign, exchange, verify"):
          self.authenticate_gradients()
      with self.tracer.span("Master: aggregated gradient computation and application"):
        if fused:
          loss_in = torch.stack([l.float().reshape(()) for l in losses]) if losses else None
          self.aggregation.step(loss_in=loss_in, prepared=True)
        else:
          self.aggregation.step(rate)
      self._refresh_weights()
    self.step += 1
    if fused:
      total = self.aggregation.loss_out[0]   # summed over workers and ranks (rank order) by the aggregation kernel: no collective here
    else:
      total = torch.stack([l.float().reshape(()) for l in losses]).sum() if losses else self._loss_buf.new_zeros(())
      if self.world > 1:
        self._loss_buf[0] = total
        dist.all_reduce(self._loss_buf, group=self.group)
        total = self._loss_buf[0]
    self.total_loss = total
    if self.debug_checksum:
      self.check_replicas()
    return total

  def evaluate(self):
    """`{"top1-X-acc": float}` on one evaluation batch, with the live parameters; under the backdoor attack, also
    `"backdoor-X-acc"`: the share of the triggered backdoor evaluation set classified as the target."""
    batch = self.experiment.eval_batch(self.device)
    metrics = self.experiment.accuracy(self.model, batch, self.eval_ctx)
    if self.backdoor_ctx is not None:
      inputs, labels = self._backdoor_batch
      metrics.update(self.experiment.backdoor_accuracy(self.model, (inputs.to(self.device), labels.to(self.device)), self.backdoor_ctx,
                                                       self.attack.target))
    return {key: float(val) for key, val in metrics.items()}

  def check_replicas(self):
    """Debug mode: every rank must hold bit-identical parameters after a step."""
    if self.device.type == "cuda":
      digest = gar_ops.checksum(self.params)
    else:
      import hashlib
      digest = torch.tensor([int.from_bytes(hashlib.blake2b(self.params.numpy().tobytes(), digest_size=7).digest(), "little")], dtype=torch.int64)
    if self.world > 1:
      gathered = [torch.zeros_like(digest) for _ in range(self.world)]
      dist.all_gather(gathered, digest, group=self.group)
      values = [int(g.item()) for g in gathered]
      if len(set(values)) != 1:
        raise RuntimeError("Replica divergence at step %d: parameter checksums %r" % (self.step, values))
    return int(digest.item())

  # ---------------------------------------------------------------------------- #
  def state_dict(self):
    """Collective when R > 1. With worker momentum, "worker_momentum" is the [n, d] fp32 matrix of every worker's momentum, indexed by
    logical worker id (n * d * 4 bytes more)."""
    agg = self.aggregation.state_dict()
    state = {"global_step": self.step, "params": self.params.detach().to("cpu", copy=True), "optimizer": self.optimizer.name,
             "aggregation": agg, "states": {k: v.detach().to("cpu", copy=True) for k, v in self.states.items()},
             "layout": self.layout.describe(), "time": time.time()}
    if self.momentum_on:
      state["worker_momentum"] = self._gather_momentum()
    return state

  def _gather_momentum(self):
    """Every rank's momentum rows -> [n, d] CPU tensor by logical worker id (collective when R > 1)."""
    if self.world > 1:
      parts = [torch.empty_like(self.worker_momentum) for _ in range(self.world)]
      dist.all_gather(parts, self.worker_momentum.contiguous(), group=self.group)
    else:
      parts = [self.worker_momentum]
    return torch.stack([parts[rank][row].detach().to("cpu", copy=True) for rank, row in self.placement])

  def load_state_dict(self, state):
    if "tf_variables" in state:  # a checkpoint of the reference: variables by name in TensorFlow's layouts, optimizer slots not carried over
      from ..tools import tf_checkpoint
      flat, states, step = tf_checkpoint.to_layout(state["tf_variables"], self.layout, self.states)
      tools.info("Imported the TensorFlow checkpoint %r (global step %s); optimizer slots start from zero" % (state.get("source", "?"), step), context="restore")
      state = {"params": flat, "states": states, "optimizer": None, "global_step": step if step is not None else 0}
    if state["params"].numel() != self.params.numel():
      raise tools.UserException("Checkpoint holds %d parameters, the model needs %d" % (state["params"].numel(), self.params.numel()))
    self.params.copy_(state["params"].to(self.device))
    for name, value in state.get("states", {}).items():
      if name in self.states:
        self.states[name].copy_(value.to(self.device))
    if state.get("optimizer") == self.optimizer.name:
      self.aggregation.load_state_dict(state["aggregation"])
    elif state.get("optimizer") is not None:
      tools.warning("Checkpoint was written with optimizer %r, now using %r: slots are reset" % (state.get("optimizer"), self.optimizer.name))
    saved = state.get("worker_momentum")
    if self.momentum_on:
      self.worker_momentum.zero_()
      if saved is None:
        tools.warning("The checkpoint holds no worker momentum: the momenta start from zero", context="restore")
      elif tuple(saved.shape) != (self.n, self.worker_momentum.shape[1]):
        raise tools.UserException("Checkpoint holds worker momenta of shape %s, expected %s" % (tuple(saved.shape), (self.n, self.worker_momentum.shape[1])))
      else:
        for i in self.local_workers:
          self.worker_momentum[self.placement[i][1]].copy_(saved[i].to(self.device))
    elif saved is not None:
      tools.warning("The checkpoint holds worker momenta but worker momentum is off: they are ignored", context="restore")
    self.step = int(state["global_step"])
    self._refresh_weights(force=True)
    if self.device.type == "cuda":
      torch.cuda.synchronize(self.device)
    if self.world > 1:
      dist.barrier(group=self.group)

  def close(self):
    if self._stream_group is not None:
      self._stream_group.close()
    if self.root_stream is not None and getattr(self.root_stream, "close", None) is not None:
      self.root_stream.close()
    for stream in self.streams:
      close = getattr(stream, "close", None)
      if close is not None:
        close()

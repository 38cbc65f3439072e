"""The parameter-server step, SPMD style: gather workers' gradients -> GAR -> optimizer -> parameters.

Three interchangeable engines share one interface (`params`, `grads`, `step()`):

* `FusedAggregation` — the product. Gradients and parameters live in symmetric (peer-mapped)
  memory; ONE cooperative sm_90a kernel per rank (`native/op_gar`) reads the owned coordinate
  slice of every worker's gradient directly from the peers over NVLink, applies the rule and the
  optimizer, and stores the new parameter slice into every rank's buffer. No NCCL call, no
  separate element-wise kernel. Each rank is a worker host *and* 1/R of the parameter server.
* `BaselineAggregation` — the "reference-style" path measured against: NCCL all-gather of the
  full flat gradients -> stand-alone GAR kernel over [n, d] -> separate optimizer kernel.
  (What `graph.py:276-281` does, with NCCL instead of gRPC.)
* `HostAggregation` — CPU tensors, gloo all-gather, host C++ GARs: the plumbing config
  (`mnist` + `average`, 2 workers) and the fallback for user plug-in GARs without a fused spec.

Logical workers: n = R * w; rank r hosts workers [r*w, (r+1)*w). The GAR always sees n rows.
Every engine also has `craft_byzantine(byz_slots, mode, coef, deviation=None, warmup=None, threshold=None, scale=None, seed=None)`, the
omniscient attacks (`attacks/omniscient.py`): the rows at the given slots of the gathered matrix are overwritten with the ALIE / IPM /
Min-Max / Min-Sum / mimic / fang-krum / fang-trim row of the others, on every rank (a collective call); `last_craft` then holds Min-Max /
Min-Sum's (gamma, A, B, C, T) of that call, fang-krum's (gamma, selected, t, gamma_max, A, B, C, T), or mimic's (s, q, ||y||^2, 1 / ||y||)
of a warm-up step. fang-krum models Krum with the engine's declared f (`f`; the number of Byzantine rows when the engine has none),
fang-trim draws with the number of the update the rows feed as step key. Mimic's state (t, z, i*; `mimic_state()`) lives in the engine (the fused
engine holds z for its owned segments only, back to back) and is checkpointed under "attack_state" as the full [d] vector.
Rules with state (`centered-clipping`: its center, `center`) keep it in the engine, and checkpoint it under "rule_state".
`dnc` draws its samples with the number of the optimizer update the aggregation feeds as step key (`updates` once it is counted,
checkpointed with it) over the padded flat size `layout.padded_size`, on every engine.
`pre_aggregation="nnm"` (nearest-neighbour mixing, `aggregators/_ops.py`) replaces every gathered row by the mean of its n - f
nearest rows before the rule runs, on every engine: inside the fused kernel, in the stand-alone kernel of the baseline engine, with
the host library's distances on the host engine and with the torch reference for plug-ins without a fused spec. The GAR object
itself does not mix. `pre_aggregation="arc"` (adaptive robust clipping) clips the k = floor(2 f (n - f) / n) rows of largest norm to
the norm of the largest row left alone, in the same places (the host engine with the torch reference); "arc+nnm" clips, then mixes.
`pre_aggregation="bucketing"` with `bucket_size` s shuffles the n gathered rows with a permutation keyed by `bucketing_seed` and the
update number (DnC's step key), and replaces them by the n' = ceil(n / s) means of buckets of s rows: the GAR is built for n' workers.
Rules that score the rows against a trusted root gradient (`fltrust`, `needs_root`) take it from `root`, a [d] fp32 row that rank 0's
trainer fills every step: the fused engine keeps it in symmetric memory and its kernel reads rank 0's copy over P2P; the baseline and
host engines broadcast it from rank 0 before the aggregation. Such rules take no pre-aggregation.
Rules with per-worker state (`foolsgold`, `needs_history`: every worker's history, the sum of the rows it submitted) keep it in the
engine as `history`, allocated with the engine (before any CUDA-graph capture) and updated by every aggregation: the baseline and host
engines hold the [n, d] fp32 matrix (every rank the whole of it), the fused engine the [n, owned] tile of its owned segments, back to
back in segment order like the staged tile, which its kernel reads and writes in place. That tile takes n * owned * 4 bytes: 0.82 GB
for ResNet-50 (d = 25 558 016) with n = 8 on one GPU, 1/R of it per rank on R ranks. The history is checkpointed under "rule_state"
as the full [n, d] CPU tensor; a checkpoint without one restores zero histories, with a warning. Such rules take no pre-aggregation:
NNM, ARC and bucketing mix, rescale or reshuffle the rows, so a row would no longer be one worker's.
"""

import os

import torch
import torch.distributed as dist

from .. import tools
from ..ops import gar as gar_ops
from .symm import SymmetricHeap


def _world(group=None):
  if dist.is_available() and dist.is_initialized():
    return dist.get_rank(group), dist.get_world_size(group)
  return 0, 1


_MIX_NAMES = {"nnm": "Nearest-neighbour mixing", "arc": "Adaptive robust clipping", "arc+nnm": "Adaptive robust clipping with nearest-neighbour mixing",
              "bucketing": "Bucketing"}


def _mixed_spec(gar, nbworkers, pre_aggregation, nb_decl_byz, bucket_size=None):
  """-> (mix, f of the mix, fused spec or None). The pre-aggregation (NNM, ARC or both) runs with the declared f: `nb_decl_byz`, or by
  default the rule's own f. Rules whose spec ignores f (average, average-nan, median, averaged-median) carry the declared f in their
  spec for the kernel's pre-aggregation. Bucketing needs no f; the GAR must have been built for the n' = ceil(n / s) bucket means."""
  from ..aggregators import FusedSpec, _ops
  mix = _ops.check_pre_aggregation(pre_aggregation, bucket_size)   # None, "nnm", "arc", "arc+nnm" or "bucketing"
  if mix is not None and getattr(gar, "needs_root", False):
    raise tools.UserException("%s scores the direction and norm of the submitted rows against the root gradient: it cannot be combined "
                              "with a pre-aggregation (got %r)" % (type(gar).__name__, mix))
  if mix is not None and getattr(gar, "needs_history", False):
    raise tools.UserException("%s keeps a history per worker: it cannot be combined with a pre-aggregation, which does not keep one row "
                              "per worker (got %r)" % (type(gar).__name__, mix))
  spec = gar.fused_spec()
  own = spec.f if spec is not None and spec.rule in FusedSpec.RULES_WITH_F else getattr(gar, "_f", None)
  f = own if nb_decl_byz is None else int(nb_decl_byz)
  if mix is None:
    return None, f, spec
  if mix == FusedSpec.BUCKETING:
    rows = _ops.check_bucketing(nbworkers, bucket_size)
    if spec is not None and spec.n != rows:
      raise tools.UserException("Bucketing with s = %d turns n = %d workers into n' = %d bucket means: the GAR must be built for %d workers (got %d)" % (
        bucket_size, nbworkers, rows, rows, spec.n))
    return mix, f, (spec.with_mix(mix, bucket_size=bucket_size) if spec is not None else None)
  name = _MIX_NAMES[mix]
  if f is None:
    raise tools.UserException(name + " needs the declared number of Byzantine workers f of GAR " + type(gar).__name__)
  if own is not None and own != f:
    raise tools.UserException(name + " runs with the rule's f = %d (got f = %d)" % (own, f))
  if not 0 <= 2 * f < nbworkers:
    raise tools.UserException(name + " needs 0 <= 2 f < n (got n = %d, f = %d)" % (nbworkers, f))
  return mix, f, (spec.with_mix(mix, f) if spec is not None else None)


class _AggregationBase:
  """Common state: layout, optimizer spec and slots, update counter."""

  def __init__(self, gar, layout, nbworkers, optimizer, group=None, pre_aggregation=None, nb_decl_byz=None, bucket_size=None, bucketing_seed=0):
    self.gar = gar
    self.mix, self.f, self.spec = _mixed_spec(gar, nbworkers, pre_aggregation, nb_decl_byz, bucket_size)
    self.bucket_size = bucket_size if self.mix == "bucketing" else None
    self.bucketing_seed = int(bucketing_seed)
    self.layout = layout
    self.n = nbworkers
    self.optimizer = optimizer
    self.group = group
    self.rank, self.world = _world(group)
    if nbworkers % self.world != 0:
      raise tools.UserException("The number of workers (%d) must be a multiple of the number of ranks (%d)" % (nbworkers, self.world))
    self.w = nbworkers // self.world
    self.d = layout.padded_size
    self.updates = 0  # number of optimizer updates applied so far
    self.slots = []
    self.center = None   # centered clipping: the rule's center v, [d] fp32
    self.attack_state = None   # mimic: {"t", "z", "istar"} (`mimic_state`)
    self.root = None   # FLTrust: the root gradient, [d] fp32, written by rank 0's trainer
    self.needs_root = bool(getattr(gar, "needs_root", False))
    self.history = None   # FoolsGold: every worker's history, [n, d] fp32 (the fused engine: [n, owned])
    self.needs_history = bool(getattr(gar, "needs_history", False))

  def _make_center(self):
    """Allocate the center (+0) when the rule is centered clipping; it lives as long as the engine and travels in checkpoints."""
    spec = self.spec
    if spec is not None and spec.rule == "centered-clipping":
      self.center = torch.zeros(self.d, dtype=torch.float32, device=self.device)

  def _make_history(self, columns):
    """Allocate the [n, columns] histories (+0) when the rule keeps one per worker; they live as long as the engine and travel in
    checkpoints."""
    if self.needs_history:
      self.history = torch.zeros((self.n, columns), dtype=torch.float32, device=self.device)

  def _broadcast_root(self):
    """The baseline and host engines: every rank takes rank 0's root row before the aggregation (collective when R > 1)."""
    if self.root is not None and self.world > 1:
      dist.broadcast(self.root, src=dist.get_global_rank(self.group, 0) if self.group is not None else 0, group=self.group)

  @property
  def first_worker(self):
    return self.rank * self.w

  def mimic_state(self):
    """Mimic's state, created at first use: t = 0, z = 1 / sqrt(d) on the real coordinates of the layout (`_ops.mimic_state`), no target."""
    if self.attack_state is None:
      from ..aggregators import _ops
      mask = self.layout.mask(self.device) if hasattr(self.layout, "mask") else torch.ones(self.d, dtype=torch.bool, device=self.device)
      packed = self._pack(mask)
      self.attack_state = _ops.mimic_state(packed.numel(), self.device, packed, real=int(mask.sum()))
    return self.attack_state

  def state_dict(self):
    state = {"updates": self.updates, "slots": [s.detach().to("cpu", copy=True) for s in self.full_slots()]}
    if self.center is not None:
      state["rule_state"] = self.full_center().detach().to("cpu", copy=True)
    if self.history is not None:
      state["rule_state"] = self.full_history().detach().to("cpu", copy=True)
    if self.attack_state is not None:
      mimic = self.attack_state
      state["attack_state"] = {"mode": "mimic", "t": int(mimic["t"]), "z": self._assemble(self._unpack(mimic["z"])).detach().to("cpu", copy=True),
                               "istar": int(mimic["istar"][0])}
    return state

  def load_state_dict(self, state):
    self.updates = int(state["updates"])
    for mine, saved in zip(self.slots, state["slots"]):
      mine.copy_(saved.to(mine.device))
    if self.center is not None:
      if state.get("rule_state") is not None:
        self.center.copy_(state["rule_state"].to(self.center.device))
      else:
        tools.warning("The checkpoint holds no center for centered clipping: it starts from zero", context="restore")
        self.center.zero_()
    if self.history is not None:
      saved = state.get("rule_state")
      if saved is not None and tuple(saved.shape) == (self.n, self.d):
        self.history.copy_(self._pack_rows(saved.to(self.device)))
      else:
        tools.warning("The checkpoint holds no [%d, %d] per-worker history: the histories start from zero" % (self.n, self.d), context="restore")
        self.history.zero_()
    if self.attack_state is not None:
      saved = state.get("attack_state")
      if saved is not None and saved.get("mode") == "mimic":
        self.attack_state["t"] = int(saved["t"])
        self.attack_state["z"].copy_(self._pack(saved["z"].to(self.device)))
        self.attack_state["istar"].fill_(int(saved["istar"]))
      else:
        tools.warning("The checkpoint holds no state for mimic: its warm-up starts again", context="restore")
        self.attack_state = None
        self.mimic_state()

  def _assemble(self, vector):
    """Full copy of a [d] vector the engine maintains (the fused engine: on the owned segments only, collective when R > 1)."""
    return vector

  def _pack(self, vector):
    """The coordinates of a [d] vector that mimic's z holds: all of them (the fused engine: its owned segments, back to back)."""
    return vector

  def _unpack(self, owned):
    """The [d] vector of `_pack`'s output (the fused engine: zero outside the owned segments)."""
    return owned

  def _pack_rows(self, matrix):
    """The columns of an [n, d] matrix that the engine's history holds: all of them (the fused engine: its owned segments)."""
    return matrix

  def _fang_kwargs(self, mode, byz_slots, threshold, scale, seed, step):
    """The keywords of a Fang attack for `craft_byzantine_` / `craft`: fang-krum's declared f and threshold, fang-trim's scale, seed and
    step key (`step`: the number of the update the crafted rows feed); none for the other attacks."""
    if mode == "fang-krum":
      return {"f": self.f if self.f is not None else len(byz_slots), "threshold": threshold}
    if mode == "fang-trim":
      return {"scale": scale, "seed": 0 if seed is None else seed, "step": step}
    return {}

  def _rule_kwargs(self):
    """Keywords of the rule's `aggregate` (and of `ops.gar.aggregate`) for the step about to be counted: centered clipping's center,
    DnC's step key."""
    if self.center is not None:
      return {"center": self.center}
    if self.root is not None:
      return {"root": self.root}
    if self.history is not None:
      return {"history": self.history}
    if self.spec is not None and self.spec.rule == "dnc":
      return {"step": self.updates + 1}
    return {}

  def _pre_aggregate(self, rows, host=False):
    """The torch reference of the pre-aggregation for the step about to be counted (bucketing: step key updates + 1)."""
    from ..aggregators import _ops
    return _ops.torch_pre_aggregate(rows, self.mix, self.f, host=host, bucket_size=self.bucket_size, seed=self.bucketing_seed, step=self.updates + 1)

  def full_slots(self):
    return self.slots

  def full_center(self):
    return self.center

  def full_history(self):
    return self.history

  # -- authentication hooks (`parallel/signing.py`) --------------------------------- #
  def visible_rows(self):
    """{worker: full flat gradient row as this rank is about to consume it}."""
    raise NotImplementedError

  def consumed_slices(self):
    """Coordinate slices (rank indices of `layout.slice_bounds`) this rank reads from every row."""
    return list(range(self.world))

  def _gather(self):
    if self.world > 1 and not self._gathered_ready:
      dist.all_gather_into_tensor(self._gathered, self.grads, group=self.group)
    self._gathered_ready = False


class HostAggregation(_AggregationBase):
  """CPU/gloo engine (also drives arbitrary `_GAR.aggregate()` plug-ins on any device)."""

  name = "host"

  def __init__(self, gar, layout, nbworkers, optimizer, group=None, device="cpu", pre_aggregation=None, nb_decl_byz=None, bucket_size=None, bucketing_seed=0):
    super().__init__(gar, layout, nbworkers, optimizer, group, pre_aggregation, nb_decl_byz, bucket_size, bucketing_seed)
    self.device = torch.device(device)
    self.params = torch.zeros(self.d, dtype=torch.float32, device=self.device)
    self.grads = torch.zeros((self.w, self.d), dtype=torch.float32, device=self.device)
    self.slots = optimizer.make_slots(self.params)
    self._make_center()
    self.root = torch.zeros(self.d, dtype=torch.float32, device=self.device) if self.needs_root else None
    self._make_history(self.d)
    self._gathered = torch.zeros((self.n, self.d), dtype=torch.float32, device=self.device) if self.world > 1 else self.grads
    self._gathered_ready = False
    self.last_aggregate = None
    self.last_craft = None   # Min-Max / Min-Sum: (gamma, A, B, C, T) of the last `craft_byzantine`; fang-krum: see the module

  def visible_rows(self):
    self._gather()
    self._gathered_ready = True
    return {i: self._gathered[i] for i in range(self.n)}

  def craft_byzantine(self, byz_slots, mode, coef, deviation=None, warmup=None, threshold=None, scale=None, seed=None):
    """Gather, then the torch reference on the gathered matrix (every rank computes the same bits)."""
    from ..aggregators import _ops
    self.visible_rows()
    fang = self._fang_kwargs(mode, byz_slots, threshold, scale, seed, self.updates + 1)
    if mode == "mimic":
      self.last_craft = _ops.torch_mimic_step_(self._gathered, byz_slots, self.mimic_state(), warmup, return_details=True)
    elif mode in _ops.OPTIMIZED_MODES or mode == "fang-krum":
      self.last_craft = _ops.torch_craft_byzantine_(self._gathered, byz_slots, mode, coef, deviation=deviation, return_details=True, **fang)
    else:
      _ops.torch_craft_byzantine_(self._gathered, byz_slots, mode, coef, **fang)

  def step(self, rate):
    self._gather()
    self._broadcast_root()
    rows = self._gathered
    if self.mix is not None:
      rows = self._pre_aggregate(rows, host=True)
    aggregated = self.gar.aggregate(rows, **self._rule_kwargs())
    self.updates += 1
    self.optimizer.apply_torch(self.params, aggregated, self.slots, rate, self.updates)
    self.last_aggregate = aggregated


class BaselineAggregation(_AggregationBase):
  """NCCL all-gather -> stand-alone GAR kernel -> separate update kernel (the baseline, not the product)."""

  name = "baseline"

  def __init__(self, gar, layout, nbworkers, optimizer, group=None, device="cuda", pre_aggregation=None, nb_decl_byz=None, bucket_size=None, bucketing_seed=0):
    super().__init__(gar, layout, nbworkers, optimizer, group, pre_aggregation, nb_decl_byz, bucket_size, bucketing_seed)
    self.device = torch.device(device)
    self.params = torch.zeros(self.d, dtype=torch.float32, device=self.device)
    self.grads = torch.zeros((self.w, self.d), dtype=torch.float32, device=self.device)
    self.slots = optimizer.make_slots(self.params)
    self._make_center()
    self.root = torch.zeros(self.d, dtype=torch.float32, device=self.device) if self.needs_root else None
    self._make_history(self.d)
    self._gathered = torch.zeros((self.n, self.d), dtype=torch.float32, device=self.device) if self.world > 1 else self.grads
    self._gathered_ready = False
    self.last_aggregate = None
    self.last_craft = None   # Min-Max / Min-Sum: (gamma, A, B, C, T) of the last `craft_byzantine`; fang-krum: see the module

  def visible_rows(self):
    self._gather()
    self._gathered_ready = True
    return {i: self._gathered[i] for i in range(self.n)}

  def craft_byzantine(self, byz_slots, mode, coef, deviation=None, warmup=None, threshold=None, scale=None, seed=None):
    """Gather, then the stand-alone crafting kernel (R = 1) on the gathered matrix (every rank computes the same bits)."""
    from ..aggregators import _ops
    self.visible_rows()
    fang = self._fang_kwargs(mode, byz_slots, threshold, scale, seed, self.updates + 1)
    if mode == "mimic":
      self.last_craft = gar_ops.craft_byzantine_(self._gathered, byz_slots, mode, state=self.mimic_state(), warmup=warmup, return_details=True)
    elif mode in _ops.OPTIMIZED_MODES or mode == "fang-krum":
      self.last_craft = gar_ops.craft_byzantine_(self._gathered, byz_slots, mode, coef, deviation=deviation, return_details=True, **fang)
    else:
      gar_ops.craft_byzantine_(self._gathered, byz_slots, mode, coef, **fang)

  def step(self, rate):
    self._gather()
    self._broadcast_root()
    state = self._rule_kwargs()
    if self.spec is not None and self.n <= gar_ops.MAX_WORKERS:
      if self.mix == "bucketing":   # the permutation's step key is DnC's
        state = dict(state, step=self.updates + 1, bucketing_seed=self.bucketing_seed)
      aggregated = gar_ops.aggregate(self.spec, self._gathered, **state)   # pre-aggregates inside the kernel
    else:
      rows = self._gathered
      if self.mix is not None:
        rows = self._pre_aggregate(rows)
      aggregated = self.gar.aggregate(rows, **state)
    self.updates += 1
    if self.optimizer.name == "sgd":
      gar_ops.sgd_(self.params, aggregated, rate)
    else:
      self.optimizer.apply_torch(self.params, aggregated, self.slots, rate, self.updates)
    self.last_aggregate = aggregated


class FusedAggregation(_AggregationBase):
  """Fused P2P gather + rule + optimizer + broadcast kernels over symmetric memory.

  `buckets`: coordinate ranges `[(lo, hi), ...]` covering the flat vector, in the order the backward pass completes them (last
  layers first). Every rank owns 1/R of EVERY bucket (its *segments*), so the distance pass of a bucket can start on all ranks as
  soon as the backward pass has produced it (`phase_a(k)`, side stream) while earlier layers are still being differentiated;
  `step()` launches the finish kernel. Without buckets a rank owns one contiguous slice (`layout.slice_bounds`).
  `device_state=True` keeps the flag epoch and the step-varying optimizer scalars in device memory (`prepare(rate)` refreshes
  them) so that the launches can be captured once in a CUDA graph; the total loss of the step comes out of the kernel
  (`loss_out`, summed over ranks in rank order): no NCCL call on the step path."""

  name = "fused"

  def __init__(self, gar, layout, nbworkers, optimizer, group=None, device="cuda", keep_aggregate=False, bf16_copy=False, max_ctas=0, buckets=None, device_state=False,
               pre_aggregation=None, nb_decl_byz=None, bucket_size=None, bucketing_seed=0):
    super().__init__(gar, layout, nbworkers, optimizer, group, pre_aggregation, nb_decl_byz, bucket_size, bucketing_seed)
    self.device = torch.device(device)
    if self.spec is None:
      raise tools.UserException("GAR " + type(gar).__name__ + " has no fused kernel; use the baseline/host engine")
    if not self.spec.gathered_rows(nbworkers):   # with bucketing `_mixed_spec` already checked n' = ceil(n / s)
      raise tools.UserException("GAR built for %d workers used with %d" % (self.spec.n, nbworkers))
    d, w, R = self.d, self.w, self.world
    self.distance_rule = self.spec.rule in ("krum", "bulyan", "mda", "smea")
    self.buckets = self._check_buckets(buckets, d)
    self.segments_of = [[self._share(lo, hi, q, R) for lo, hi in self.buckets] for q in range(R)]
    self.segments = self.segments_of[self.rank]
    self.lo, self.hi = self.segments[0][0], self.segments[-1][1]   # meaningful for a single bucket (contiguous slice)
    owned = sum(hi - lo for lo, hi in self.segments)
    signal_bytes, mailbox_bytes = gar_ops.region_bytes()
    sizes = {"grads": w * d * 4, "params": d * 4, "signals": signal_bytes, "mailbox": mailbox_bytes}
    if bf16_copy:
      sizes["params_bf16"] = d * 2
    if self.needs_root:
      sizes["root"] = d * 4
    self.heap = SymmetricHeap(SymmetricHeap.required(*sizes.values()), self.device, group)
    for name, nbytes in sizes.items():
      self.heap.region(name, nbytes)
    self.grads = self.heap.local("grads", torch.float32, (w, d))
    self.params = self.heap.local("params", torch.float32)
    self.params_bf16 = self.heap.local("params_bf16", torch.bfloat16) if bf16_copy else None
    self.root = self.heap.local("root", torch.float32) if self.needs_root else None   # only rank 0's copy is read
    self.slots = optimizer.make_slots(self.params)
    self._make_center()   # centered clipping: maintained on the owned segments only, like the optimizer slots
    self._make_history(owned)   # FoolsGold: the owned segments of every worker's history, back to back
    self.aggregate_out = torch.zeros(d, dtype=torch.float32, device=self.device) if keep_aggregate else None
    # staging keeps the P2P-loaded tiles local so that later passes never cross NVLink again (and rows beyond the 8 held in registers
    # can be re-read); needed whenever the distance pass and the aggregation pass are different launches too
    # the iterative rules' passes after the first re-read the staged copy rather than the peers' rows; a pre-aggregation (NNM mixes, ARC
    # clips) rewrites the staged tile in place and every rule then reads it (n * owned * 4 bytes, also with R = 1); bucketing stores its
    # n' means there, so the tile has the rule's spec.n rows
    # FLTrust's and FoolsGold's second pass reads the staged rows over several ranks, and beyond one 8-row block
    need_staging = ((self.distance_rule and (R > 1 or len(self.buckets) > 1 or self.n > 8)) or (self.spec.rule in gar_ops.ITERATIVE_RULES and R > 1)
                    or self.mix is not None or (self.spec.rule in ("fltrust", "foolsgold") and (R > 1 or self.n > 8)))
    self.staging = torch.empty((self.spec.n, owned), dtype=torch.float32, device=self.device) if need_staging else None
    self.launcher = gar_ops.FusedLauncher(self.device, self.n)
    if self.spec.rule == "dnc":
      self.launcher.dnc_scratch(self.spec, d)   # allocated before any graph capture
    if self.spec.rule == "smea":
      self.launcher.smea_scratch(self.spec)
    self.max_ctas = max_ctas
    self.epoch = 0
    self.device_state = bool(device_state)
    self.epoch_dev = torch.zeros(1, dtype=torch.int32, device=self.device) if device_state else None
    self.hyper_dev = torch.zeros(4, dtype=torch.float32, device=self.device) if device_state else None
    self._hyper_host = torch.zeros(4, dtype=torch.float32).pin_memory() if device_state else None
    keyed = self.spec.rule == "dnc" or self.mix == "bucketing"
    # DnC, bucketing: the step key of the samples and of the permutation, refreshed by `prepare` so that graph replays draw new ones
    self.step_dev = torch.zeros(1, dtype=torch.int64, device=self.device) if device_state and keyed else None
    self.loss_out = torch.zeros(1, dtype=torch.float32, device=self.device)
    self._pre_accumulated = 0
    self._craft_mode = None   # Min-Max / Min-Sum: (mode, H) of the last `craft_byzantine`
    self._prepared = False   # `prepare` ran for the step that has not been aggregated yet
    self._row_views = None
    heap = self.heap
    self._rows = [heap.peer(i // w, "grads") + (i % w) * d * 4 for i in range(self.n)]
    self._param_dst = [heap.peer(q, "params") for q in range(R)]
    self._param_bf16_dst = [heap.peer(q, "params_bf16") for q in range(R)] if bf16_copy else None
    self._signals = [heap.peer(q, "signals") for q in range(R)]
    self._mailboxes = [heap.peer(q, "mailbox") for q in range(R)]
    self._root_src = heap.peer(0, "root") if self.needs_root else None
    self._param_mc = heap.multicast("params") if R > 1 else 0
    # in-switch (NVLS) reduction of the gradients for the `average` rule instead of 7 P2P loads (0.241 vs 0.312 ms at 8 GPUs); AGB_NVLS_REDUCE=0 disables
    self._grad_mc = heap.multicast("grads") if (R > 1 and self.spec.rule == "average" and self.mix is None and os.environ.get("AGB_NVLS_REDUCE", "1") not in ("", "0")) else 0
    tools.info("Fused aggregation: rule %r%s, n = %d (%d per rank), d = %d, %d bucket(s), %d owned coordinates, provider %s, NVLS multicast %s" % (
      self.spec.rule, {"nnm": " after NNM", "arc": " after ARC", "arc+nnm": " after ARC and NNM", "bucketing": " after bucketing (s = %s)" % self.bucket_size}.get(self.mix, ""), self.n, w, d, len(self.buckets), owned, heap.provider, "on" if self._param_mc else "off"), context="fused")

  @staticmethod
  def _check_buckets(buckets, d):
    if not buckets:
      return [(0, d)]
    buckets = [(int(lo), int(hi)) for lo, hi in buckets]
    if len(buckets) > gar_ops.MAX_SEGMENTS:
      raise tools.UserException("At most %d gradient buckets" % gar_ops.MAX_SEGMENTS)
    covered = sorted(buckets)
    if covered[0][0] != 0 or covered[-1][1] != d or any(a[1] != b[0] for a, b in zip(covered, covered[1:])) or any(lo % 4 or hi % 4 or hi <= lo for lo, hi in covered):
      raise tools.UserException("Gradient buckets must tile [0, d) with bounds that are multiples of 4: " + repr(buckets))
    return buckets

  @staticmethod
  def _share(lo, hi, rank, world):
    quads = (hi - lo) // 4
    return lo + (quads * rank // world) * 4, lo + (quads * (rank + 1) // world) * 4

  @property
  def last_aggregate(self):
    return self.aggregate_out

  @property
  def overlappable(self):
    """Whether `phase_a` exists for this rule (the distance pass of Krum / Bulyan / MDA / SMEA is additive over coordinates); not with a
    pre-aggregation, whose first pass (NNM's raw distances, ARC's norms, bucketing's means) runs in the finish kernel over every segment."""
    return self.distance_rule and len(self.buckets) > 1 and self.mix is None

  def visible_rows(self):
    """Every worker's row through the peer mapping — the very addresses the fused kernel dereferences."""
    if self._row_views is None:
      from .symm import _view
      self._row_views = {}
      for i in range(self.n):
        if i // self.w == self.rank:
          self._row_views[i] = self.grads[i % self.w]
        else:
          self._row_views[i] = _view(self._rows[i], self.d * 4, self.device, self.heap).view(torch.float32)
    return self._row_views

  def consumed_slices(self):
    return [self.rank]

  def _common(self, rate_args):
    lr, hyper = rate_args
    return dict(opt=self.optimizer.name, lr=lr, hyper=hyper, param=self.params, slot0=self.slots[0] if len(self.slots) > 0 else None,
                slot1=self.slots[1] if len(self.slots) > 1 else None, param_dst=self._param_dst, param_mc=self._param_mc, param_bf16_dst=self._param_bf16_dst,
                rank=self.rank, R=self.world, signals=self._signals, mailboxes=self._mailboxes, staging=self.staging, max_ctas_limit=self.max_ctas,
                grad_mc=self._grad_mc, workers_per_rank=self.w, row_stride=self.d, epoch_ptr=self.epoch_dev, hyper_ptr=self.hyper_dev)

  def prepare(self, rate):
    """Host side of one step: advance the update counter and (device-state mode) refresh the device copy of the optimizer scalars.
    Stream-ordered before the kernels of the step; never part of a captured graph."""
    self.updates += 1
    self.epoch += 1
    self._prepared = True
    self._rate_args = self.optimizer.kernel_args(rate, self.updates)
    if self.device_state:
      lr, hyper = self._rate_args
      self._hyper_host[0], self._hyper_host[1], self._hyper_host[2], self._hyper_host[3] = lr, hyper[0], hyper[1], hyper[2]
      self.hyper_dev.copy_(self._hyper_host, non_blocking=True)
      if self.step_dev is not None:   # the value travels as a kernel argument of the fill, fixed when it is enqueued
        self.step_dev.fill_(self.updates)

  def craft_byzantine(self, byz_slots, mode, coef, stream=None, deviation=None, warmup=None, threshold=None, scale=None, seed=None):
    """Collective: this rank crafts its owned segments of every Byzantine row, local or on a peer (`ops.gar.craft`), behind an entry
    barrier at the epoch of the step about to be aggregated. Every rank calls it, including ranks that host no Byzantine worker.
    Min-Max / Min-Sum and fang-krum exchange their statistics through the mailboxes; `last_craft` reads gamma and the sums back (a
    synchronisation). Mimic's warm-up steps exchange theirs the same way and update z on the owned segments."""
    from ..aggregators import _ops
    byz_slots = _ops.check_byzantine_slots(self.n, byz_slots, mode)
    optimized = mode in _ops.OPTIMIZED_MODES or mode == "fang-krum"
    mimic = mode == "mimic"
    if mode in _ops.OPTIMIZED_MODES:
      deviation = _ops.check_deviation(mode, deviation)
    state = None
    if mimic:
      warmup = _ops.check_mimic(self.n, byz_slots, warmup)[1]
      state = self.mimic_state()
      warm = state["t"] < warmup
    epoch = self.epoch if self._prepared else self.epoch + 1
    fang = self._fang_kwargs(mode, byz_slots, threshold, scale, seed, self.updates if self._prepared else self.updates + 1)
    gar_ops.craft(self._rows, self.segments, [i for i in range(self.n) if i not in byz_slots], byz_slots, mode, coef, deviation=deviation,
                  launcher=self.launcher if optimized or mimic else None, mailboxes=self._mailboxes if optimized or mimic else None, R=self.world,
                  rank=self.rank, signals=self._signals, epoch=epoch, epoch_ptr=self.epoch_dev, stream=stream, state=state, warmup=warmup, **fang)
    self._craft_mode = (mode, self.n - len(byz_slots)) if optimized or (mimic and warm) else None

  @property
  def last_craft(self):
    """Min-Max / Min-Sum: (gamma, A, B, C, T) of the last `craft_byzantine`, as the kernel solved them (identical on every rank); fang-krum:
    (gamma, selected, t, gamma_max, A, B, C, T); mimic: (s, q, ||y||^2, 1 / ||y||) of the last call when it was a warm-up step."""
    mode = self._craft_mode
    if mode is not None and mode[0] == "mimic":
      return gar_ops.mimic_details(self.launcher, mode[1])
    if mode is not None and mode[0] == "fang-krum":
      return gar_ops.fang_krum_details(self.launcher, mode[1])
    return None if mode is None else gar_ops.craft_details(self.launcher, *mode)

  def phase_a(self, seg, stream=None):
    """Distance pass + staging of bucket `seg` (buckets must be pre-accumulated in order 0, 1, ...). Call between `prepare` and `step`."""
    if seg != self._pre_accumulated:
      raise AssertionError("buckets are pre-accumulated in order")
    self.launcher.phase_a(self.spec, self._rows, self.segments, seg, stream=stream, epoch=self.epoch, first_seg=seg + 1, **self._common(self._rate_args))
    self._pre_accumulated = seg + 1

  def step(self, rate=None, stream=None, loss_in=None, prepared=False):
    """The finish kernel. `rate` is ignored when `prepare(rate)` was already called for this step (`prepared=True`)."""
    if not prepared:
      self.prepare(rate)
    self._prepared = False
    first_seg, self._pre_accumulated = self._pre_accumulated, 0
    self.launcher.launch(self.spec, self._rows, segments=self.segments, agg_out=self.aggregate_out, epoch=self.epoch, stream=stream, first_seg=first_seg,
                         loss_in=loss_in, loss_out=self.loss_out, center=self.center, step=self.updates, step_ptr=self.step_dev, domain=self.d,
                         bucketing_seed=self.bucketing_seed, root=self._root_src, history=self.history, **self._common(self._rate_args))

  def _assemble(self, vector):
    """Full copy of a [d] vector maintained on the owned segments only (collective when R > 1)."""
    if self.world == 1:
      return vector
    merged = vector.clone()
    for q in range(self.world):
      for lo, hi in self.segments_of[q]:
        if hi == lo:
          continue
        piece = merged[lo:hi].contiguous() if q == self.rank else torch.empty(hi - lo, dtype=vector.dtype, device=vector.device)
        dist.broadcast(piece, src=dist.get_global_rank(self.group, q) if self.group is not None else q, group=self.group)
        merged[lo:hi] = piece
    return merged

  def full_slots(self):
    """Optimizer slots are only maintained on the owned segments: assemble the full vectors (checkpoints)."""
    if self.world == 1 or not self.slots:
      return self.slots
    return [self._assemble(slot) for slot in self.slots]

  def full_center(self):
    """The center of centered clipping, assembled from the owned segments of every rank (checkpoints)."""
    return None if self.center is None else self._assemble(self.center)

  def full_history(self):
    """FoolsGold's [n, d] histories, assembled from the owned segments of every rank (checkpoints; collective when R > 1)."""
    if self.history is None:
      return None
    return torch.stack([self._assemble(self._unpack(row)) for row in self.history])

  def _pack_rows(self, matrix):
    return torch.cat([matrix[:, lo:hi] for lo, hi in self.segments], dim=1)

  def _pack(self, vector):
    """Mimic's z and y scratch hold the owned segments only, back to back in segment order (as the staged tile): d / R floats each."""
    return torch.cat([vector[lo:hi] for lo, hi in self.segments])

  def _unpack(self, owned):
    full = torch.zeros(self.d, dtype=owned.dtype, device=owned.device)
    at = 0
    for lo, hi in self.segments:
      full[lo:hi] = owned[at:at + hi - lo]
      at += hi - lo
    return full


def _single_host(group=None):
  """Whether every rank of the group runs on the same machine (collective call). Peer-mapped memory — hence the fused engine —
  only exists inside one NVLink domain; ranks spread over several hosts (deploy.py over SSH) go through NCCL."""
  if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
    return True
  import socket
  hosts = [None] * dist.get_world_size(group)
  dist.all_gather_object(hosts, socket.gethostname(), group=group)
  return len(set(hosts)) == 1


def make_aggregation(kind, gar, layout, nbworkers, optimizer, group=None, device="cpu", pre_aggregation=None, nb_decl_byz=None, bucket_size=None,
                     bucketing_seed=0, **kwargs):
  """`kind` in {"auto", "fused", "baseline", "host"}; "auto" = fused on CUDA when the rule has a kernel and all ranks share one
  machine, the NCCL baseline engine on CUDA otherwise, host on CPU. `pre_aggregation`: None / "none", "nnm", "arc" or "arc+nnm", on every engine, with
  `nb_decl_byz` declared Byzantine workers (default: the rule's f), or "bucketing" with `bucket_size` and `bucketing_seed`."""
  mix = dict(pre_aggregation=pre_aggregation, nb_decl_byz=nb_decl_byz, bucket_size=bucket_size, bucketing_seed=bucketing_seed)
  device = torch.device(device)
  if kind == "auto":
    if device.type != "cuda":
      kind = "host"
    elif gar.fused_spec() is not None and nbworkers <= gar_ops.MAX_WORKERS:
      kind = "fused"
      if not _single_host(group):
        tools.warning("The ranks span several hosts: no peer-mapped memory between them, using the NCCL all-gather engine", context="fused")
        kind = "baseline"
    else:
      kind = "baseline"
  if kind == "fused":
    return FusedAggregation(gar, layout, nbworkers, optimizer, group, device, **mix, **kwargs)
  if kind == "baseline":
    return BaselineAggregation(gar, layout, nbworkers, optimizer, group, device, **mix)
  if kind == "host":
    return HostAggregation(gar, layout, nbworkers, optimizer, group, device, **mix)
  raise tools.UserException("Unknown aggregation engine " + repr(kind))

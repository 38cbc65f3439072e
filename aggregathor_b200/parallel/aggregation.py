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
Every engine also has `craft_byzantine(byz_slots, mode, coef)`, the omniscient attacks (`attacks/omniscient.py`): the rows at the
given slots of the gathered matrix are overwritten with the ALIE / IPM row of the others, on every rank (a collective call).
Rules with state (`centered-clipping`: its center, `center`) keep it in the engine, and checkpoint it under "rule_state".
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


class _AggregationBase:
  """Common state: layout, optimizer spec and slots, update counter."""

  def __init__(self, gar, layout, nbworkers, optimizer, group=None):
    self.gar = gar
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

  def _make_center(self):
    """Allocate the center (+0) when the rule is centered clipping; it lives as long as the engine and travels in checkpoints."""
    spec = self.gar.fused_spec()
    if spec is not None and spec.rule == "centered-clipping":
      self.center = torch.zeros(self.d, dtype=torch.float32, device=self.device)

  @property
  def first_worker(self):
    return self.rank * self.w

  def state_dict(self):
    state = {"updates": self.updates, "slots": [s.detach().to("cpu", copy=True) for s in self.full_slots()]}
    if self.center is not None:
      state["rule_state"] = self.full_center().detach().to("cpu", copy=True)
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

  def full_slots(self):
    return self.slots

  def full_center(self):
    return self.center

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

  def __init__(self, gar, layout, nbworkers, optimizer, group=None, device="cpu"):
    super().__init__(gar, layout, nbworkers, optimizer, group)
    self.device = torch.device(device)
    self.params = torch.zeros(self.d, dtype=torch.float32, device=self.device)
    self.grads = torch.zeros((self.w, self.d), dtype=torch.float32, device=self.device)
    self.slots = optimizer.make_slots(self.params)
    self._make_center()
    self._gathered = torch.zeros((self.n, self.d), dtype=torch.float32, device=self.device) if self.world > 1 else self.grads
    self._gathered_ready = False
    self.last_aggregate = None

  def visible_rows(self):
    self._gather()
    self._gathered_ready = True
    return {i: self._gathered[i] for i in range(self.n)}

  def craft_byzantine(self, byz_slots, mode, coef):
    """Gather, then the torch reference on the gathered matrix (every rank computes the same bits)."""
    from ..aggregators import _ops
    self.visible_rows()
    _ops.torch_craft_byzantine_(self._gathered, byz_slots, mode, coef)

  def step(self, rate):
    self._gather()
    aggregated = self.gar.aggregate(self._gathered) if self.center is None else self.gar.aggregate(self._gathered, center=self.center)
    self.updates += 1
    self.optimizer.apply_torch(self.params, aggregated, self.slots, rate, self.updates)
    self.last_aggregate = aggregated


class BaselineAggregation(_AggregationBase):
  """NCCL all-gather -> stand-alone GAR kernel -> separate update kernel (the baseline, not the product)."""

  name = "baseline"

  def __init__(self, gar, layout, nbworkers, optimizer, group=None, device="cuda"):
    super().__init__(gar, layout, nbworkers, optimizer, group)
    self.device = torch.device(device)
    self.spec = gar.fused_spec()
    self.params = torch.zeros(self.d, dtype=torch.float32, device=self.device)
    self.grads = torch.zeros((self.w, self.d), dtype=torch.float32, device=self.device)
    self.slots = optimizer.make_slots(self.params)
    self._make_center()
    self._gathered = torch.zeros((self.n, self.d), dtype=torch.float32, device=self.device) if self.world > 1 else self.grads
    self._gathered_ready = False
    self.last_aggregate = None

  def visible_rows(self):
    self._gather()
    self._gathered_ready = True
    return {i: self._gathered[i] for i in range(self.n)}

  def craft_byzantine(self, byz_slots, mode, coef):
    """Gather, then the stand-alone crafting kernel on the gathered matrix (every rank computes the same bits)."""
    self.visible_rows()
    gar_ops.craft_byzantine_(self._gathered, byz_slots, mode, coef)

  def step(self, rate):
    self._gather()
    state = {} if self.center is None else {"center": self.center}
    if self.spec is not None and self.n <= gar_ops.MAX_WORKERS:
      aggregated = gar_ops.aggregate(self.spec, self._gathered, **state)
    else:
      aggregated = self.gar.aggregate(self._gathered, **state)
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

  def __init__(self, gar, layout, nbworkers, optimizer, group=None, device="cuda", keep_aggregate=False, bf16_copy=False, max_ctas=0, buckets=None, device_state=False):
    super().__init__(gar, layout, nbworkers, optimizer, group)
    self.device = torch.device(device)
    self.spec = gar.fused_spec()
    if self.spec is None:
      raise tools.UserException("GAR " + type(gar).__name__ + " has no fused kernel; use the baseline/host engine")
    if self.spec.n != nbworkers:
      raise tools.UserException("GAR built for %d workers used with %d" % (self.spec.n, nbworkers))
    d, w, R = self.d, self.w, self.world
    self.distance_rule = self.spec.rule in ("krum", "bulyan", "mda")
    self.buckets = self._check_buckets(buckets, d)
    self.segments_of = [[self._share(lo, hi, q, R) for lo, hi in self.buckets] for q in range(R)]
    self.segments = self.segments_of[self.rank]
    self.lo, self.hi = self.segments[0][0], self.segments[-1][1]   # meaningful for a single bucket (contiguous slice)
    owned = sum(hi - lo for lo, hi in self.segments)
    sizes = {"grads": w * d * 4, "params": d * 4, "signals": gar_ops.SIGNAL_BYTES, "mailbox": gar_ops.MAILBOX_BYTES}
    if bf16_copy:
      sizes["params_bf16"] = d * 2
    self.heap = SymmetricHeap(SymmetricHeap.required(*sizes.values()), self.device, group)
    for name, nbytes in sizes.items():
      self.heap.region(name, nbytes)
    self.grads = self.heap.local("grads", torch.float32, (w, d))
    self.params = self.heap.local("params", torch.float32)
    self.params_bf16 = self.heap.local("params_bf16", torch.bfloat16) if bf16_copy else None
    self.slots = optimizer.make_slots(self.params)
    self._make_center()   # centered clipping: maintained on the owned segments only, like the optimizer slots
    self.aggregate_out = torch.zeros(d, dtype=torch.float32, device=self.device) if keep_aggregate else None
    # staging keeps the P2P-loaded tiles local so that later passes never cross NVLink again (and rows beyond the 8 held in registers
    # can be re-read); needed whenever the distance pass and the aggregation pass are different launches too
    # the iterative rules' passes after the first re-read the staged copy rather than the peers' rows
    need_staging = (self.distance_rule and (R > 1 or len(self.buckets) > 1 or self.n > 8)) or (self.spec.rule in gar_ops.ITERATIVE_RULES and R > 1)
    self.staging = torch.empty((self.n, owned), dtype=torch.float32, device=self.device) if need_staging else None
    self.launcher = gar_ops.FusedLauncher(self.device, self.n)
    self.max_ctas = max_ctas
    self.epoch = 0
    self.device_state = bool(device_state)
    self.epoch_dev = torch.zeros(1, dtype=torch.int32, device=self.device) if device_state else None
    self.hyper_dev = torch.zeros(4, dtype=torch.float32, device=self.device) if device_state else None
    self._hyper_host = torch.zeros(4, dtype=torch.float32).pin_memory() if device_state else None
    self.loss_out = torch.zeros(1, dtype=torch.float32, device=self.device)
    self._pre_accumulated = 0
    self._prepared = False   # `prepare` ran for the step that has not been aggregated yet
    self._row_views = None
    heap = self.heap
    self._rows = [heap.peer(i // w, "grads") + (i % w) * d * 4 for i in range(self.n)]
    self._param_dst = [heap.peer(q, "params") for q in range(R)]
    self._param_bf16_dst = [heap.peer(q, "params_bf16") for q in range(R)] if bf16_copy else None
    self._signals = [heap.peer(q, "signals") for q in range(R)]
    self._mailboxes = [heap.peer(q, "mailbox") for q in range(R)]
    self._param_mc = heap.multicast("params") if R > 1 else 0
    # in-switch (NVLS) reduction of the gradients for the `average` rule instead of 7 P2P loads (0.241 vs 0.312 ms at 8 GPUs); AGB_NVLS_REDUCE=0 disables
    self._grad_mc = heap.multicast("grads") if (R > 1 and self.spec.rule == "average" and os.environ.get("AGB_NVLS_REDUCE", "1") not in ("", "0")) else 0
    tools.info("Fused aggregation: rule %r, n = %d (%d per rank), d = %d, %d bucket(s), %d owned coordinates, provider %s, NVLS multicast %s" % (
      self.spec.rule, self.n, w, d, len(self.buckets), owned, heap.provider, "on" if self._param_mc else "off"), context="fused")

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
    """Whether `phase_a` exists for this rule (the distance pass of Krum / Bulyan / MDA is additive over coordinates)."""
    return self.distance_rule and len(self.buckets) > 1

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

  def craft_byzantine(self, byz_slots, mode, coef, stream=None):
    """Collective: this rank crafts its owned segments of every Byzantine row, local or on a peer (`ops.gar.craft`), behind an entry
    barrier at the epoch of the step about to be aggregated. Every rank calls it, including ranks that host no Byzantine worker."""
    from ..aggregators import _ops
    byz_slots = _ops.check_byzantine_slots(self.n, byz_slots, mode)
    epoch = self.epoch if self._prepared else self.epoch + 1
    gar_ops.craft(self._rows, self.segments, [i for i in range(self.n) if i not in byz_slots], byz_slots, mode, coef, R=self.world, rank=self.rank,
                  signals=self._signals, epoch=epoch, epoch_ptr=self.epoch_dev, stream=stream)

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
                         loss_in=loss_in, loss_out=self.loss_out, center=self.center, **self._common(self._rate_args))

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


def _single_host(group=None):
  """Whether every rank of the group runs on the same machine (collective call). Peer-mapped memory — hence the fused engine —
  only exists inside one NVLink domain; ranks spread over several hosts (deploy.py over SSH) go through NCCL."""
  if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
    return True
  import socket
  hosts = [None] * dist.get_world_size(group)
  dist.all_gather_object(hosts, socket.gethostname(), group=group)
  return len(set(hosts)) == 1


def make_aggregation(kind, gar, layout, nbworkers, optimizer, group=None, device="cpu", **kwargs):
  """`kind` in {"auto", "fused", "baseline", "host"}; "auto" = fused on CUDA when the rule has a kernel and all ranks share one
  machine, the NCCL baseline engine on CUDA otherwise, host on CPU."""
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
    return FusedAggregation(gar, layout, nbworkers, optimizer, group, device, **kwargs)
  if kind == "baseline":
    return BaselineAggregation(gar, layout, nbworkers, optimizer, group, device)
  if kind == "host":
    return HostAggregation(gar, layout, nbworkers, optimizer, group, device)
  raise tools.UserException("Unknown aggregation engine " + repr(kind))

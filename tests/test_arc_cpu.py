"""Adaptive robust clipping (ARC) on the CPU: the clip count, the factors on hand-built norms (ties at the threshold, C = +0, a
non-finite threshold, clipped infinite and NaN norms), properties on random rows with outliers, the host engine against the torch
reference for every rule with "arc" and "arc+nnm", the option checks, and short training runs under attack."""

import math

import numpy as np
import pytest
import torch

from aggregathor_b200 import aggregators, attacks, experiments, tools
from aggregathor_b200.aggregators import FusedSpec, _ops
from aggregathor_b200.cli import runner
from aggregathor_b200.engine.flat import FlatLayout
from aggregathor_b200.engine.optimizers import optimizers
from aggregathor_b200.engine.schedules import build
from aggregathor_b200.engine.trainer import Manager
from aggregathor_b200.parallel.aggregation import HostAggregation, make_aggregation

U = 2.0 ** -24
INF, NAN = float("inf"), float("nan")


def _equal_bits(a, b):
  a, b = torch.as_tensor(a).cpu(), torch.as_tensor(b).cpu()
  assert a.dtype == b.dtype and a.shape == b.shape
  nan = torch.isnan(a)
  assert torch.equal(nan, torch.isnan(b))
  assert torch.equal(a[~nan].view(torch.int32), b[~nan].view(torch.int32))


def _f32(value):
  return float(np.float32(value))


@pytest.mark.parametrize("n,f,k", [(1, 0, 0), (2, 0, 0), (3, 1, 1), (5, 2, 2), (8, 2, 3), (9, 4, 4), (11, 2, 3), (17, 5, 7), (32, 7, 10),
                                   (32, 15, 15), (7, 0, 0)])
def test_clip_count(n, f, k):
  assert _ops.arc_clip_count(n, f) == k == (2 * f * (n - f)) // n


def test_invalid_parameters():
  for n, f in ((4, 2), (3, 2), (1, 1), (5, -1)):
    with pytest.raises(tools.UserException, match="2 f < n"):
      _ops.arc_clip_count(n, f)
    with pytest.raises(tools.UserException):
      _ops.torch_arc(torch.randn(n, 10), f)
  for name in ("arc", "arc+nnm"):
    assert _ops.check_pre_aggregation(name) == name
  for name in ("bucketing", "nnm+arc", "clip"):
    with pytest.raises(tools.UserException):
      _ops.check_pre_aggregation(name)


def _factors(values, f):
  c, clipped = _ops.arc_factors(torch.tensor(values, dtype=torch.float32), f)
  assert c.dtype == torch.float32 and clipped.dtype == torch.bool
  return c.tolist(), [i for i in range(len(values)) if bool(clipped[i])]


def test_factors_ties_at_the_threshold():
  # n = 8, f = 2: k = 3; ascending order rows 6, 0, 1, 7, 2 | 3, 4, 5: the threshold is row 2 (N = 4, C = 2) and the three clipped
  # rows tie with it, so their factor is exactly 1
  c, clipped = _factors([1.0, 2.0, 4.0, 4.0, 4.0, 4.0, 0.5, 3.0], 2)
  assert clipped == [3, 4, 5] and c == [1.0] * 8
  # a clipped row just above the threshold is scaled
  c, clipped = _factors([1.0, 2.0, 4.0, 4.0, 4.0, 9.0, 0.5, 3.0], 2)
  assert clipped == [3, 4, 5] and c[3] == c[4] == 1.0 and c[5] == _f32(2.0 / 3.0)


def test_factors_threshold_zero():
  c, clipped = _factors([0.0, 0.0, 4.0], 1)   # n = 3, f = 1: k = 1, C = sqrt(0) = +0
  assert clipped == [2] and c == [1.0, 1.0, 0.0] and math.copysign(1.0, c[2]) == 1.0
  c, clipped = _factors([0.0, 0.0, 0.0], 1)   # the clipped row ties with C = +0: s <= C, factor 1 (no 0 / 0)
  assert clipped == [2] and c == [1.0, 1.0, 1.0]


def test_factors_non_finite_threshold():
  # n = 8, f = 2: k = 3, but four norms are not finite: the threshold row (position 4) is one of them, nothing is clipped
  c, clipped = _factors([1.0, INF, NAN, 2.0, INF, 3.0, NAN, 4.0], 2)
  assert clipped == [] and c == [1.0] * 8
  # f = 0: k = 0, nothing is clipped whatever the norms
  c, clipped = _factors([1.0, INF, 1e30, NAN], 0)
  assert clipped == [] and c == [1.0] * 4


def test_factors_clipped_infinite_and_nan_norms():
  # ascending: rows 0, 1, 2, 3, 4 (C = sqrt(5)), then 7 (N = 6), 5 (+inf), 6 (NaN): the last three are clipped
  c, clipped = _factors([1.0, 2.0, 3.0, 4.0, 5.0, INF, NAN, 6.0], 2)
  assert clipped == [5, 6, 7]
  C, s7 = _f32(math.sqrt(5.0)), _f32(math.sqrt(6.0))
  assert c[:5] == [1.0] * 5 and c[7] == float(np.float32(C) / np.float32(s7))
  assert c[5] == 0.0 and math.isnan(c[6])
  G = torch.ones(8, 4)
  G[5, 1] = INF
  G[6, 2] = NAN
  factors = torch.tensor(c, dtype=torch.float32)
  Y = _ops.torch_arc_clip(G, factors)
  assert bool(torch.isnan(Y[5, 1])) and torch.equal(Y[5, [0, 2, 3]], torch.zeros(3))   # inf * 0 is NaN, 1 * 0 is 0
  assert bool(torch.isnan(Y[6]).all())
  _equal_bits(Y[:5], G[:5])


def _rows(n, d, seed, outliers=0, non_finite=False):
  """Small-integer rows (every squared norm is an exact fp32 integer): honest rows in [-4, 4], outliers scaled by 20."""
  gen = torch.Generator().manual_seed(seed)
  G = torch.randint(-4, 5, (n, d), generator=gen).float()
  for k in range(outliers):
    G[n - 1 - k] = G[n - 1 - k] * 20
  if non_finite:
    G[0, 3::11] = NAN
    G[1, 5] = INF
  return G


@pytest.mark.parametrize("n,f", [(3, 1), (5, 2), (8, 2), (9, 4), (17, 5), (32, 7)])
def test_properties_on_rows_with_outliers(n, f):
  d = 301
  G = _rows(n, d, seed=7 * n + f, outliers=f)
  Y, N, c, clipped = _ops.torch_arc(G, f, return_details=True)
  k = _ops.arc_clip_count(n, f)
  exact = (G.double() ** 2).sum(dim=1)
  assert torch.equal(N.double(), exact)   # exact integers in fp32
  order = sorted(range(n), key=lambda i: (float(N[i]), i))
  assert [i for i in range(n) if bool(clipped[i])] == sorted(order[n - k:])
  C = _f32(math.sqrt(float(N[order[n - k - 1]])))
  for i in range(n):
    if not bool(clipped[i]):
      _equal_bits(Y[i], G[i])   # unclipped rows are bit-identical
      assert float(c[i]) == 1.0
      continue
    x, y = G[i].double(), Y[i].double()
    assert math.sqrt(float((y * y).sum())) <= C * (1 + 4 * U)
    if float(c[i]) != 1.0:   # parallel: y = c x up to one rounding per element
      assert float((y - float(c[i]) * x).abs().max()) <= U * float(y.abs().max())
      assert float((y * x).sum()) > 0
  # the f outliers are the largest rows, so they are among the clipped ones
  assert all(bool(clipped[n - 1 - j]) for j in range(f))


def test_f_zero_is_the_identity():
  G = _rows(7, 503, seed=3, outliers=2)
  _equal_bits(_ops.torch_arc(G, 0), G)
  G[2, 4] = NAN
  _equal_bits(_ops.torch_arc(G, 0), G)


def test_non_finite_rows_are_clipped_last():
  G = _rows(9, 301, seed=5, outliers=1, non_finite=True)
  Y, N, c, clipped = _ops.torch_arc(G, 2, return_details=True)   # k = 3: rows 1 (inf), 0 (NaN) and the outlier
  assert [i for i in range(9) if bool(clipped[i])] == [0, 1, 8]
  assert math.isnan(float(c[0])) and float(c[1]) == 0.0 and 0.0 < float(c[8]) < 1.0
  assert bool(torch.isnan(Y[0]).all()) and bool(torch.isnan(Y[1, 5])) and float(Y[1].nan_to_num().abs().max()) == 0.0


def test_spec_ids_and_repr():
  spec = FusedSpec("krum", 8, f=2, m=3)
  assert FusedSpec.MIXES == (None, "nnm", "arc", "arc+nnm")
  assert [spec.with_mix(mix).mix_id for mix in FusedSpec.MIXES] == [0, 1, 2, 3]
  assert repr(spec) == "FusedSpec(rule='krum', n=8, f=2, m=3, beta=0)"
  assert repr(spec.with_mix("nnm")) == "FusedSpec(rule='krum', n=8, f=2, m=3, beta=0, mix='nnm')"
  assert repr(spec.with_mix("arc")) == "FusedSpec(rule='krum', n=8, f=2, m=3, beta=0, mix='arc')"
  assert repr(spec.with_mix("arc+nnm")) == "FusedSpec(rule='krum', n=8, f=2, m=3, beta=0, mix='arc+nnm')"
  with pytest.raises(tools.UserException):
    FusedSpec("krum", 8, f=2, mix="nnm+arc")


def test_pre_aggregate_composes_arc_then_nnm():
  G = _rows(9, 401, seed=11, outliers=2)
  _equal_bits(_ops.torch_pre_aggregate(G, None, 2), G)
  _equal_bits(_ops.torch_pre_aggregate(G, "arc", 2), _ops.torch_arc(G, 2))
  _equal_bits(_ops.torch_pre_aggregate(G, "nnm", 2), _ops.torch_nnm(G, 2))
  _equal_bits(_ops.torch_pre_aggregate(G, "arc+nnm", 2), _ops.torch_nnm(_ops.torch_arc(G, 2), 2))
  _equal_bits(_ops.torch_pre_aggregate(G, "arc+nnm", 2, host=True), _ops.host_nnm(_ops.torch_arc(G, 2), 2))


RULES = [("average", []), ("average-nan", []), ("median", []), ("averaged-median", []), ("krum", []), ("bulyan", []), ("trimmed-mean", []),
         ("mda", []), ("geometric-median", ["iterations:3"]), ("centered-clipping", ["iterations:2", "tau:2"]),
         ("dnc", ["iterations:2", "subsample:300"])]


def _layout(d):
  layout = FlatLayout()
  layout.add("theta", (d,))
  layout.freeze()
  return layout


def _randn_rows(n, d, seed, outliers):
  gen = torch.Generator().manual_seed(seed)
  G = torch.randn(n, d, generator=gen)
  for k in range(outliers):
    G[n - 1 - k] = G[n - 1 - k] * 30 + 5
  return G


@pytest.mark.parametrize("mix", ["arc", "arc+nnm"])
@pytest.mark.parametrize("rule,args", RULES, ids=[r for r, _ in RULES])
def test_host_engine_matches_the_torch_reference(rule, args, mix):
  n, f, d = 11, 2, 1003
  gar = aggregators.instantiate(rule, n, f, args)
  layout = _layout(d)
  engine = HostAggregation(gar, layout, n, build(optimizers, "optimizer", "sgd", []), pre_aggregation=mix, nb_decl_byz=f)
  assert engine.mix == mix and engine.f == f and engine.spec.mix == mix
  center = torch.zeros(layout.padded_size)
  for step in range(2):
    G = torch.zeros(n, layout.padded_size)
    G[:, :d] = _randn_rows(n, d, seed=10 * step + len(rule), outliers=f)
    engine.grads.copy_(G)
    engine.step(0.1)
    Y = _ops.torch_arc(G, f)
    if mix == "arc+nnm":
      Y = _ops.torch_nnm(Y, f)
    state = {"center": center} if rule == "centered-clipping" else {"step": step + 1} if rule == "dnc" else {}
    expect = gar.aggregate(Y, **state)
    _equal_bits(engine.last_aggregate, expect)
    if rule == "average":   # the clip changed what the rule saw
      assert not torch.equal(gar.aggregate(G), expect)
  if rule == "centered-clipping":
    _equal_bits(engine.center, center)


def test_engine_options():
  layout = _layout(64)
  sgd = build(optimizers, "optimizer", "sgd", [])
  gar = aggregators.instantiate("average", 5, 0, [])
  with pytest.raises(tools.UserException, match="Adaptive robust clipping"):   # average keeps no f: ARC needs the declared one
    make_aggregation("host", gar, layout, 5, sgd, pre_aggregation="arc")
  engine = make_aggregation("host", gar, layout, 5, sgd, pre_aggregation="arc", nb_decl_byz=2)
  assert engine.spec.mix == "arc" and engine.spec.f == 2 and engine.spec.mix_id == 2 and gar.fused_spec().mix is None
  for mix in ("arc", "arc+nnm"):
    with pytest.raises(tools.UserException, match="2 f < n"):
      make_aggregation("host", gar, layout, 5, sgd, pre_aggregation=mix, nb_decl_byz=3)
  krum = aggregators.instantiate("krum", 7, 2, [])
  with pytest.raises(tools.UserException):   # ARC runs with the rule's own f
    make_aggregation("host", krum, layout, 7, sgd, pre_aggregation="arc", nb_decl_byz=1)
  engine = make_aggregation("host", krum, layout, 7, sgd, pre_aggregation="arc+nnm")
  assert engine.f == 2 and engine.spec.mix_id == 3


def test_runner_options():
  base = ["--client", "x", "--experiment", "mnist", "--aggregator", "median", "--nb-workers", "5"]
  for mix in ("arc", "arc+nnm"):
    args = runner.make_parser().parse_args(base + ["--pre-aggregation", mix, "--nb-decl-byz-workers", "2"])
    assert args.pre_aggregation == mix
    runner._validate(args)
    for f in ("3", "-1"):
      args = runner.make_parser().parse_args(base + ["--pre-aggregation", mix, "--nb-decl-byz-workers", f])
      with pytest.raises(tools.UserException, match="2 f < n"):
        runner._validate(args)
  with pytest.raises(SystemExit):
    runner.make_parser().parse_args(base + ["--pre-aggregation", "nnm+arc"])


def _manager(gar_name, n, f, attack=None, real=0, args=(), attack_args=(), seed=0, **kwargs):
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate(gar_name, n, f, list(args))
  attack = attacks.instantiate(attack, n, f, list(attack_args)) if attack else None
  return Manager(experiment, gar, n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu", attack=attack, nb_real_byz=real, seed=seed,
                 **kwargs)


def test_arc_off_is_bit_identical_to_no_option():
  plain = _manager("median", 3, 1)
  off = _manager("median", 3, 1, pre_aggregation="none", nb_decl_byz=1)
  assert off.aggregation.mix is None and off.pre_aggregation is None
  for _ in range(3):
    plain.train()
    off.train()
  _equal_bits(plain.params, off.params)


def test_arc_bounds_a_scaled_flip_attack():
  # average over n = 8 workers, 2 of them submitting -1e6 times their gradient: without ARC the step is dominated by the attackers
  # and the loss blows up; with ARC their rows are clipped to an honest-sized norm
  n, f, steps = 8, 2, 6
  runs = {}
  for mix in ("none", "arc"):
    mgr = _manager("average", n, f, "flip", f, attack_args=["factor:-1e6"], seed=3, pre_aggregation=mix, nb_decl_byz=f)
    losses = [float(mgr.train()) for _ in range(steps)]
    runs[mix] = (losses, mgr.params.clone())
  arc_losses, arc_params = runs["arc"]
  plain_losses, plain_params = runs["none"]
  assert bool(torch.isfinite(arc_params).all()) and all(math.isfinite(v) for v in arc_losses)
  # with this seed the unclipped run diverges: from the second step on its loss explodes, then its parameters turn NaN
  assert plain_losses[1] > 1e6 * plain_losses[0] and not bool(torch.isfinite(plain_params).all())
  # with ARC the loss (summed over the 8 workers) still goes down
  assert arc_losses[-1] < arc_losses[0] and max(arc_losses) <= arc_losses[0]


@pytest.mark.parametrize("mix", ["arc", "arc+nnm"])
def test_training_with_momentum_under_alie(mix):
  n, f = 7, 2
  mgr = _manager("trimmed-mean", n, f, "alie", f, worker_momentum=0.9, worker_momentum_dampening=0.1, pre_aggregation=mix, nb_decl_byz=f)
  assert mgr.aggregation.mix == mix
  start = mgr.params.clone()
  for _ in range(3):
    assert bool(torch.isfinite(mgr.train()))
  assert bool(torch.isfinite(mgr.params).all()) and not torch.equal(mgr.params, start)

"""Nearest-neighbour mixing (NNM) on the CPU: selection and mixing against a NumPy fp32 transcription of the definition, ties and
non-finite rows, f = 0, the host engine against the torch reference for every rule, training with NNM under attacks, and the option
checks."""

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


def _equal_bits(a, b):
  a, b = torch.as_tensor(a).cpu(), torch.as_tensor(b).cpu()
  assert a.dtype == b.dtype and a.shape == b.shape
  nan = torch.isnan(a)
  assert torch.equal(nan, torch.isnan(b))
  assert torch.equal(a[~nan].view(torch.int32), b[~nan].view(torch.int32))


def _np_select(D, f):
  """N_i: i and the n - f - 1 other rows first by (finite ascending, non-finite last, lower index on ties)."""
  n = D.shape[0]
  member = np.zeros((n, n), dtype=bool)
  for i in range(n):
    key = lambda j: (0, float(D[i, j]), j) if np.isfinite(D[i, j]) else (1, 0.0, j)
    others = sorted((j for j in range(n) if j != i), key=key)
    member[i, i] = True
    member[i, others[:n - f - 1]] = True
  return member


def _np_mix(X, member, f):
  """y_i = (((x_a0 + x_a1) + ...) / (n - f) in NumPy fp32, members in ascending order from +0."""
  n = X.shape[0]
  Y = np.empty_like(X)
  with np.errstate(over="ignore", invalid="ignore"):
    for i in range(n):
      s = np.zeros(X.shape[1], dtype=np.float32)
      for j in range(n):
        if member[i, j]:
          s = s + X[j]
      Y[i] = s / np.float32(n - f)
  return Y


def _rows(n, d, seed, outliers=0, non_finite=False):
  gen = torch.Generator().manual_seed(seed)
  G = torch.randn(n, d, generator=gen)
  for k in range(outliers):
    G[n - 1 - k] = G[n - 1 - k] * 30 + 5
  if non_finite:
    G[0, 3::11] = float("nan")
    G[1, 5] = float("inf")
  return G


@pytest.mark.parametrize("n,f", [(3, 1), (5, 2), (8, 2), (9, 4), (17, 5), (32, 7)])
def test_select_and_mix_match_numpy(n, f):
  G = _rows(n, 301, seed=n + f, outliers=f, non_finite=n >= 8)
  dist = _ops.torch_pairwise_distances(G)
  member = _ops.nnm_select(dist, f)
  assert torch.equal(member, torch.from_numpy(_np_select(dist.numpy(), f)))
  assert bool(member.diagonal().all()) and (member.sum(dim=1) == n - f).all()
  Y = _ops.torch_nnm_mix(G, member, f)
  _equal_bits(Y, torch.from_numpy(_np_mix(G.numpy(), member.numpy(), f)))
  _equal_bits(_ops.torch_nnm_mix(G, _ops.nnm_bits(member), f), Y)   # the kernel's bit masks select the same rows
  _equal_bits(_ops.torch_nnm(G, f), Y)
  if n >= 8:   # a row with a NaN is in its own neighbourhood: its mix is NaN
    assert bool(torch.isnan(Y[0]).any())


def test_ties_and_non_finite_distances():
  n, f = 6, 2
  inf = float("inf")
  D = torch.zeros(n, n)
  # rows 0, 1, 2 are duplicates (distance 0); row 5 has non-finite distances to everyone
  D[:3, :3] = 0.0
  for i, j, v in ((0, 3, 4.0), (0, 4, 4.0), (1, 3, 1.0), (1, 4, 9.0), (2, 3, 2.0), (2, 4, 2.0), (3, 4, 3.0)):
    D[i, j] = D[j, i] = v
  D[5, :5] = D[:5, 5] = inf
  D[0, 5] = D[5, 0] = float("nan")
  member = _ops.nnm_select(D, f)
  assert torch.equal(member, torch.from_numpy(_np_select(D.numpy(), f)))
  rows = lambda i: [j for j in range(n) if bool(member[i, j])]
  assert rows(0) == [0, 1, 2, 3]    # the two duplicates first, then the lower index of the tie 3 / 4 at 4.0
  assert rows(1) == [0, 1, 2, 3]
  assert rows(2) == [0, 1, 2, 3]    # duplicates at distance 0 tie with each other: lower indices first, itself regardless
  assert rows(5) == [0, 1, 2, 5]    # all its distances are non-finite: the lowest indices, and itself
  assert rows(4) == [0, 2, 3, 4]    # 2.0 (j = 2) first, 3.0 (j = 3), then 4.0 (j = 0) before 9.0 (j = 1)
  # a row whose distances are all non-finite still mixes with itself first, whatever its index
  D2 = torch.full((3, 3), inf).fill_diagonal_(0.0)
  assert [j for j in range(3) if bool(_ops.nnm_select(D2, 1)[2, j])] == [0, 2]


def test_f_zero_mixes_every_row_into_the_mean():
  G = _rows(7, 503, seed=3, outliers=2)
  Y = _ops.torch_nnm(G, 0)
  total = torch.zeros(503)
  for i in range(7):
    total = total + G[i]
  mean = total / torch.tensor(7.0)
  for i in range(7):
    _equal_bits(Y[i], mean)


def test_invalid_parameters():
  for n, f in ((4, 2), (3, 2), (1, 1), (5, -1)):
    with pytest.raises(tools.UserException):
      _ops.check_nnm(n, f)
  with pytest.raises(tools.UserException):
    _ops.torch_nnm(torch.randn(4, 10), 2)
  with pytest.raises(tools.UserException):
    _ops.check_pre_aggregation("bucketing")
  assert _ops.check_pre_aggregation("none") is None and _ops.check_pre_aggregation("nnm") == "nnm"
  with pytest.raises(tools.UserException):
    FusedSpec("krum", 8, f=2, mix="bucketing")
  spec = FusedSpec("krum", 8, f=2, m=3)
  mixed = spec.with_mix("nnm")
  assert repr(spec) == "FusedSpec(rule='krum', n=8, f=2, m=3, beta=0)" and repr(mixed) == "FusedSpec(rule='krum', n=8, f=2, m=3, beta=0, mix='nnm')"
  assert spec.mix_id == 0 and mixed.mix_id == 1 and spec.mix is None


RULES = [("average", []), ("average-nan", []), ("median", []), ("averaged-median", []), ("krum", []), ("bulyan", []), ("trimmed-mean", []),
         ("mda", []), ("geometric-median", ["iterations:3"]), ("centered-clipping", ["iterations:2", "tau:2"])]


def _layout(d):
  layout = FlatLayout()
  layout.add("theta", (d,))
  layout.freeze()
  return layout


@pytest.mark.parametrize("rule,args", RULES, ids=[r for r, _ in RULES])
def test_host_engine_matches_the_torch_reference(rule, args):
  n, f, d = 11, 2, 1003
  gar = aggregators.instantiate(rule, n, f, args)
  layout = _layout(d)
  engine = HostAggregation(gar, layout, n, build(optimizers, "optimizer", "sgd", []), pre_aggregation="nnm", nb_decl_byz=f)
  assert engine.mix == "nnm" and engine.f == f
  center = torch.zeros(layout.padded_size)
  for step in range(2):
    G = torch.zeros(n, layout.padded_size)
    G[:, :d] = _rows(n, d, seed=10 * step + len(rule), outliers=f)
    engine.grads.copy_(G)
    engine.step(0.1)
    dist = _ops.torch_pairwise_distances(G)
    assert torch.equal(_ops.nnm_select(_ops.host_pairwise_distances(G), f), _ops.nnm_select(dist, f))
    Y = _ops.torch_nnm(G, f)
    expect = gar.aggregate(Y, center=center) if rule == "centered-clipping" else gar.aggregate(Y)
    _equal_bits(engine.last_aggregate, expect)
    plain = gar.aggregate(G, center=center.clone()) if rule == "centered-clipping" else gar.aggregate(G)
    assert not torch.equal(plain, expect)   # the mix changed what the rule saw
  if rule == "centered-clipping":
    _equal_bits(engine.center, center)


def test_engine_options():
  layout = _layout(64)
  sgd = build(optimizers, "optimizer", "sgd", [])
  gar = aggregators.instantiate("average", 5, 0, [])
  with pytest.raises(tools.UserException):   # average keeps no f: NNM needs the declared one
    make_aggregation("host", gar, layout, 5, sgd, pre_aggregation="nnm")
  engine = make_aggregation("host", gar, layout, 5, sgd, pre_aggregation="nnm", nb_decl_byz=2)
  assert engine.spec.mix == "nnm" and engine.spec.f == 2 and gar.fused_spec().mix is None
  assert make_aggregation("host", gar, layout, 5, sgd).spec.mix is None
  with pytest.raises(tools.UserException):   # 2 f >= n
    make_aggregation("host", gar, layout, 5, sgd, pre_aggregation="nnm", nb_decl_byz=3)
  krum = aggregators.instantiate("krum", 7, 2, [])
  with pytest.raises(tools.UserException):   # NNM runs with the rule's own f
    make_aggregation("host", krum, layout, 7, sgd, pre_aggregation="nnm", nb_decl_byz=1)
  assert make_aggregation("host", krum, layout, 7, sgd, pre_aggregation="nnm").f == 2


def _manager(gar_name, n, f, attack=None, real=0, args=(), **kwargs):
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate(gar_name, n, f, list(args))
  return Manager(experiment, gar, n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu", attack=attack, nb_real_byz=real, **kwargs)


@pytest.mark.parametrize("attack", ["alie", "flip"])
@pytest.mark.parametrize("rule,args", [("trimmed-mean", []), ("krum", []), ("centered-clipping", ["iterations:2", "tau:1"])])
def test_training_with_nnm_under_attack(rule, args, attack):
  n, f = 7, 2
  mgr = _manager(rule, n, f, attacks.instantiate(attack, n, f, []), f, args=args, worker_momentum=0.9, worker_momentum_dampening=0.1,
                 pre_aggregation="nnm", nb_decl_byz=f)
  assert mgr.aggregation.mix == "nnm"
  start = mgr.params.clone()
  for _ in range(3):
    loss = mgr.train()
    assert bool(torch.isfinite(loss))
  assert bool(torch.isfinite(mgr.params).all()) and not torch.equal(mgr.params, start)


def test_nnm_off_is_bit_identical_to_no_option():
  plain = _manager("median", 3, 1)
  off = _manager("median", 3, 1, pre_aggregation="none", nb_decl_byz=1)
  assert off.aggregation.mix is None and off.pre_aggregation is None
  for _ in range(3):
    plain.train()
    off.train()
  _equal_bits(plain.params, off.params)


def test_runner_options():
  base = ["--client", "x", "--experiment", "mnist", "--aggregator", "median", "--nb-workers", "5"]
  args = runner.make_parser().parse_args(base)
  assert args.pre_aggregation == "none"
  args = runner.make_parser().parse_args(base + ["--pre-aggregation", "nnm", "--nb-decl-byz-workers", "2"])
  assert args.pre_aggregation == "nnm"
  runner._validate(args)
  with pytest.raises(SystemExit):
    runner.make_parser().parse_args(base + ["--pre-aggregation", "bucketing"])
  for f in ("3", "-1"):
    args = runner.make_parser().parse_args(base + ["--pre-aggregation", "nnm", "--nb-decl-byz-workers", f])
    with pytest.raises(tools.UserException, match="2 f < n"):
      runner._validate(args)
  args = runner.make_parser().parse_args(base + ["--nb-decl-byz-workers", "3"])
  runner._validate(args)   # without NNM, 2 f >= n only warns
  with pytest.raises(tools.UserException):
    _manager("median", 4, 2, pre_aggregation="nnm", nb_decl_byz=2)


def test_deploy_forwards_the_option():
  from aggregathor_b200.cli import deploy
  cmd = deploy.rank_command(["--pre-aggregation", "nnm"], False)
  assert cmd[-2:] == ["--pre-aggregation", "nnm"]

"""Bucketing on the CPU: the keyed permutation (against pinned values of an independent transcription of its definition), the bucket
masks, the bucket means against a NumPy float32 oracle bit for bit (NaN and infinities included), the host engine against the torch
reference for every rule valid at n', the option checks, a short training run under ALIE and a checkpoint resume."""

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

INF, NAN = float("inf"), float("nan")
M64 = (1 << 64) - 1


def _equal_bits(a, b):
  a, b = torch.as_tensor(a).cpu(), torch.as_tensor(b).cpu()
  assert a.dtype == b.dtype and a.shape == b.shape
  nan = torch.isnan(a)
  assert torch.equal(nan, torch.isnan(b))
  assert torch.equal(a[~nan].view(torch.int32), b[~nan].view(torch.int32))


# ---------------------------------------------------------------------------- #
# An independent transcription of the definition: NumPy uint64 arithmetic (wrapping), no shared code with `_ops`

def _mix64(z):
  with np.errstate(over="ignore"):
    z = np.uint64(z) + np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def _oracle_permutation(n, seed, step):
  key = _mix64(_mix64(_mix64(np.uint64(seed)) ^ np.uint64(step)) ^ np.uint64(_ops.BUCKETING_TAG))
  perm = list(range(n))
  for i in range(n - 1, 0, -1):
    j = int(_mix64(key ^ np.uint64(i)) % np.uint64(i + 1))
    perm[i], perm[j] = perm[j], perm[i]
  return perm


def _oracle_means(X, s, perm):
  """NumPy float32: members of every bucket added in ascending worker order from +0, then one division."""
  n = X.shape[0]
  out = []
  for b in range(-(-n // s)):
    members = sorted(perm[b * s:min((b + 1) * s, n)])
    acc = np.zeros(X.shape[1], dtype=np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
      for j in members:
        acc = (acc + X[j]).astype(np.float32)
      out.append((acc / np.float32(len(members))).astype(np.float32))
  return torch.from_numpy(np.stack(out))


# ---------------------------------------------------------------------------- #
# Permutation and masks

def test_tag_differs_from_dnc_iteration_keys():
  assert _ops.BUCKETING_TAG >= 8 > _ops.DNC_MAX_ITERATIONS - 1


@pytest.mark.parametrize("n", [1, 2, 3, 8, 9, 17, 32, 45])
def test_permutation_is_a_permutation_and_matches_the_oracle(n):
  for seed in (0, 1, 12345, M64):
    for step in (0, 1, 2, 7, 1 << 40, (1 << 63) - 1):
      perm = _ops.bucketing_permutation(n, seed, step)
      assert sorted(perm) == list(range(n))
      assert perm == _oracle_permutation(n, seed, step)


# values of the transcription above, written down once: a change of the key, the tag or the shuffle shows here
PINNED = {(8, 0, 1): [4, 0, 3, 5, 7, 2, 6, 1],
          (16, 3, 5): [1, 11, 15, 8, 2, 14, 0, 5, 12, 7, 6, 9, 3, 13, 10, 4],
          (32, M64, 123456789): [22, 20, 31, 5, 19, 18, 8, 3, 10, 0, 4, 26, 2, 12, 15, 13, 27, 11, 17, 1, 25, 21, 28, 14, 30, 24, 23, 29, 9, 7,
                                 6, 16]}


def test_pinned_permutations():
  for (n, seed, step), perm in PINNED.items():
    assert _ops.bucketing_permutation(n, seed, step) == perm == _oracle_permutation(n, seed, step)


def test_permutation_changes_with_step_and_seed():
  n = 16
  perms = {tuple(_ops.bucketing_permutation(n, 0, step)) for step in range(1, 21)}
  assert len(perms) == 20
  assert _ops.bucketing_permutation(n, 0, 1) != _ops.bucketing_permutation(n, 1, 1)


@pytest.mark.parametrize("n,s", [(1, 1), (3, 1), (3, 2), (3, 3), (8, 2), (8, 3), (9, 2), (9, 4), (17, 3), (17, 17), (32, 2), (32, 5)])
def test_masks_partition_the_rows(n, s):
  perm = _ops.bucketing_permutation(n, 4, 9)
  masks = _ops.bucketing_masks(n, s, perm)
  assert len(masks) == _ops.check_bucketing(n, s) == math.ceil(n / s)
  union = 0
  for b, mask in enumerate(masks):
    assert union & mask == 0
    union |= mask
    size = bin(mask).count("1")
    assert size == (s if b < len(masks) - 1 else n - s * (len(masks) - 1))
    assert mask == sum(1 << perm[p] for p in range(b * s, min((b + 1) * s, n)))
  assert union == (1 << n) - 1


def test_one_bucket_and_singleton_buckets():
  gen = torch.Generator().manual_seed(1)
  G = torch.randn(7, 33, generator=gen)
  G[2, 4] = -0.0
  one = _ops.torch_bucketing(G, 7, 0, 3)
  assert one.shape == (1, 33)
  _equal_bits(one[0], _oracle_means(G.numpy(), 7, list(range(7)))[0])
  Y, perm, masks = _ops.torch_bucketing(G, 1, 0, 3, return_details=True)
  perm = perm.tolist()
  expect = G[perm].clone()
  expect[expect == 0] = 0.0   # -0 becomes +0 (+0 + -0 = +0)
  _equal_bits(Y, expect)
  assert masks.tolist() == [1 << p for p in perm]


# ---------------------------------------------------------------------------- #
# Bucket means

def _rows(n, d, seed, non_finite=False):
  gen = torch.Generator().manual_seed(seed)
  G = torch.randn(n, d, generator=gen) * torch.logspace(-3, 3, d)
  if non_finite and n >= 3:
    G[0, 1] = NAN
    G[1, 2] = INF
    G[2, 2] = -INF   # +inf and -inf in a bucket give NaN, alone they stay infinite
    G[n - 1, 5] = INF
  G[n // 2, 0] = -0.0
  return G


@pytest.mark.parametrize("non_finite", [False, True])
@pytest.mark.parametrize("n,s", [(3, 2), (8, 2), (8, 3), (9, 2), (17, 3), (32, 2), (32, 32)])
def test_means_match_the_numpy_oracle_bit_for_bit(n, s, non_finite):
  G = _rows(n, 257, seed=n * 31 + s, non_finite=non_finite)
  for step in (1, 2):
    Y, perm, masks = _ops.torch_bucketing(G, s, 11, step, return_details=True)
    assert perm.dtype == torch.int32 and masks.dtype == torch.int32
    assert perm.tolist() == _oracle_permutation(n, 11, step)
    _equal_bits(Y, _oracle_means(G.numpy(), s, perm.tolist()))


def test_pre_aggregate_dispatch():
  G = _rows(9, 40, seed=2)
  _equal_bits(_ops.torch_pre_aggregate(G, "bucketing", None, bucket_size=2, seed=5, step=4), _ops.torch_bucketing(G, 2, 5, 4))
  _equal_bits(_ops.torch_pre_aggregate(G, None, 2, bucket_size=2), G)


# ---------------------------------------------------------------------------- #
# Engines

RULES = [("average", []), ("average-nan", []), ("median", []), ("averaged-median", []), ("krum", []), ("bulyan", []), ("trimmed-mean", []),
         ("mda", []), ("geometric-median", ["iterations:3"]), ("centered-clipping", ["iterations:2", "tau:2"]),
         ("dnc", ["iterations:2", "subsample:300"]), ("smea", [])]


def _layout(d):
  layout = FlatLayout()
  layout.add("theta", (d,))
  layout.freeze()
  return layout


def _valid(rule, rows, f):
  try:
    aggregators.instantiate(rule, rows, f, [])
    return True
  except tools.UserException:
    return False


@pytest.mark.parametrize("n,s,f", [(11, 2, 1), (16, 2, 1), (9, 3, 0)])
@pytest.mark.parametrize("rule,args", RULES, ids=[r for r, _ in RULES])
def test_host_engine_matches_the_torch_reference(rule, args, n, s, f):
  rows = math.ceil(n / s)
  if not _valid(rule, rows, f):
    pytest.skip("%s is not valid at n' = %d, f = %d" % (rule, rows, f))
  d = 301
  gar = aggregators.instantiate(rule, rows, f, args)
  layout = _layout(d)
  engine = HostAggregation(gar, layout, n, build(optimizers, "optimizer", "sgd", []), pre_aggregation="bucketing", bucket_size=s,
                           bucketing_seed=7)
  assert engine.mix == "bucketing" and engine.bucket_size == s
  assert engine.spec.mix == "bucketing" and engine.spec.n == rows and engine.spec.mix_id == FusedSpec.MIX_BUCKETING
  center = torch.zeros(layout.padded_size)
  for step in range(2):
    G = torch.zeros(n, layout.padded_size)
    G[:, :d] = _rows(n, d, seed=10 * step + len(rule))
    engine.grads.copy_(G)
    engine.step(0.1)
    Y = _ops.torch_bucketing(G, s, 7, step + 1)
    state = {"center": center} if rule == "centered-clipping" else {"step": step + 1} if rule == "dnc" else {}
    _equal_bits(engine.last_aggregate, gar.aggregate(Y, **state))


def test_spec_and_option_checks():
  spec = FusedSpec("krum", 4, f=1, m=1)
  assert FusedSpec.MIXES == (None, "nnm", "arc", "arc+nnm")   # bucketing is not one of the NNM / ARC bit combinations
  bucketed = spec.with_mix("bucketing", bucket_size=2)
  assert bucketed.mix_id == 4 and bucketed.bucket_size == 2 and bucketed.gathered_rows(8) and bucketed.gathered_rows(7)
  assert not bucketed.gathered_rows(9) and not bucketed.gathered_rows(4)
  assert repr(bucketed) == "FusedSpec(rule='krum', n=4, f=1, m=1, beta=0, mix='bucketing', bucket_size=2)"
  for size in (None, 0, -1, 1.5, True):
    with pytest.raises(tools.UserException, match="bucket size"):
      FusedSpec("krum", 4, f=1, mix="bucketing", bucket_size=size)
  with pytest.raises(tools.UserException, match="bucket size"):
    _ops.check_pre_aggregation("bucketing")
  assert _ops.check_pre_aggregation("bucketing", 2) == "bucketing"
  for n, s in ((4, 0), (4, 5), (1, 2), (4, -1)):
    with pytest.raises(tools.UserException, match="1 <= s <= n"):
      _ops.check_bucketing(n, s)
  with pytest.raises(tools.UserException):
    _ops.bucketing_permutation(4, -1, 1)
  with pytest.raises(tools.UserException):
    _ops.bucketing_permutation(4, 0, -1)


def test_engine_options():
  layout = _layout(64)
  sgd = build(optimizers, "optimizer", "sgd", [])
  average4 = aggregators.instantiate("average", 4, 0, [])
  engine = make_aggregation("host", average4, layout, 8, sgd, pre_aggregation="bucketing", bucket_size=2)
  assert engine.spec.n == 4 and engine.spec.bucket_size == 2 and average4.fused_spec().mix is None
  for s in (0, 9):   # s out of range
    with pytest.raises(tools.UserException, match="1 <= s <= n"):
      make_aggregation("host", average4, layout, 8, sgd, pre_aggregation="bucketing", bucket_size=s)
  with pytest.raises(tools.UserException, match="bucket size"):
    make_aggregation("host", average4, layout, 8, sgd, pre_aggregation="bucketing")
  average8 = aggregators.instantiate("average", 8, 0, [])   # built for n instead of n'
  with pytest.raises(tools.UserException, match=r"n = 8 workers into n' = 4 bucket means"):
    make_aggregation("host", average8, layout, 8, sgd, pre_aggregation="bucketing", bucket_size=2)
  for combined in ("bucketing+nnm", "arc+bucketing", "nnm+bucketing"):   # not a pre-aggregation: bucketing is never combined
    with pytest.raises(tools.UserException, match="Unknown pre-aggregation"):
      make_aggregation("host", average4, layout, 8, sgd, pre_aggregation=combined, bucket_size=2)
  for mix in ("nnm", "arc"):
    with pytest.raises(tools.UserException):
      FusedSpec("krum", 4, f=1, mix=mix + "+bucketing", bucket_size=2)


def test_runner_options():
  base = ["--client", "x", "--experiment", "mnist", "--aggregator", "krum", "--nb-workers", "8", "--nb-decl-byz-workers", "2"]
  with pytest.raises(SystemExit):   # bucketing is only complete with its bucket size
    runner.make_parser().parse_args(base + ["--pre-aggregation", "bucketing"])
  args = runner.make_parser().parse_args(base + ["--pre-aggregation", "bucketing", "--bucket-size", "2"])
  assert args.pre_aggregation == "bucketing" and args.bucket_size == 2 and runner.make_parser().parse_args(base).bucket_size is None
  runner._validate(args)
  # Krum with n = 8, s = 2, f = 2: n' = 4 < f + 3, the rule's own message with the n -> n' context
  with pytest.raises(tools.UserException, match=r"(?s)Krum.*n = 8 workers into n' = 4 bucket means"):
    runner._instantiate_aggregator(args, 8)
  args = runner.make_parser().parse_args(base + ["--pre-aggregation", "bucketing", "--bucket-size", "1"])
  runner._validate(args)
  assert runner._instantiate_aggregator(args, 8).fused_spec().n == 8
  for s in ("0", "9"):
    args = runner.make_parser().parse_args(base + ["--pre-aggregation", "bucketing", "--bucket-size", s])
    with pytest.raises(tools.UserException, match="1 <= s <= n"):
      runner._validate(args)
  with pytest.raises(SystemExit):
    runner.make_parser().parse_args(base + ["--pre-aggregation", "bucketing+nnm"])


# ---------------------------------------------------------------------------- #
# Training

def _manager(gar_name, n, f, rows, attack=None, real=0, args=(), seed=0, **kwargs):
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate(gar_name, rows, f, list(args))
  attack = attacks.instantiate(attack, n, f, []) if attack else None
  return Manager(experiment, gar, n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu", attack=attack, nb_real_byz=real, seed=seed,
                 **kwargs)


def test_training_under_alie_decreases_the_loss():
  n, f, s = 8, 1, 2
  mgr = _manager("trimmed-mean", n, f, 4, "alie", f, seed=5, pre_aggregation="bucketing", bucket_size=s, bucketing_seed=5)
  assert mgr.aggregation.mix == "bucketing" and mgr.aggregation.spec.n == 4
  losses = [float(mgr.train()) for _ in range(6)]
  assert all(math.isfinite(v) for v in losses) and bool(torch.isfinite(mgr.params).all())
  assert losses[-1] < losses[0]


def test_checkpoint_resume_follows_the_update_count():
  layout = _layout(50)
  gar = aggregators.instantiate("median", 3, 0, [])
  gen = torch.Generator().manual_seed(21)
  grads = [torch.randn(6, layout.padded_size, generator=gen) for _ in range(5)]

  def engine():
    return HostAggregation(gar, layout, 6, build(optimizers, "optimizer", "sgd", []), pre_aggregation="bucketing", bucket_size=2,
                           bucketing_seed=9)
  straight = engine()
  for G in grads:
    straight.grads.copy_(G)
    straight.step(0.1)
  first = engine()
  for G in grads[:2]:
    first.grads.copy_(G)
    first.step(0.1)
  resumed = engine()
  resumed.params.copy_(first.params)
  resumed.load_state_dict(first.state_dict())
  for G in grads[2:]:
    resumed.grads.copy_(G)
    resumed.step(0.1)
  _equal_bits(resumed.params, straight.params)
  # a resume that forgot the update count draws other permutations
  fresh = engine()
  fresh.params.copy_(first.params)
  for G in grads[2:]:
    fresh.grads.copy_(G)
    fresh.step(0.1)
  assert not torch.equal(fresh.params, straight.params)

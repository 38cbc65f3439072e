"""SMEA (smallest maximum eigenvalue averaging) on the CPU: the vectorised scores against `dnc_eigh` set by set, the selection against a
float64 covariance oracle, planted cases, the selection keys, the host engine against the torch reference with every pre-aggregation,
argument checks and a seeded mnist run under ALIE."""

import itertools
import math

import numpy as np
import pytest
import torch

from aggregathor_b200 import aggregators, attacks, experiments, tools
from aggregathor_b200.aggregators import FusedSpec, _ops
from aggregathor_b200.engine.flat import FlatLayout
from aggregathor_b200.engine.optimizers import optimizers
from aggregathor_b200.engine.schedules import build
from aggregathor_b200.engine.trainer import Manager
from aggregathor_b200.parallel.aggregation import HostAggregation

U = 2.0 ** -24


def _equal_bits(a, b):
  a, b = a.cpu(), b.cpu()
  assert a.dtype == b.dtype and a.shape == b.shape
  nan = torch.isnan(a)
  assert torch.equal(nan, torch.isnan(b))
  assert torch.equal(a[~nan].view(torch.int32) if a.dtype == torch.float32 else a[~nan], b[~nan].view(torch.int32) if b.dtype == torch.float32 else b[~nan])


def _per_set_scores(dist, f):
  """The score of every kept set, one `dnc_eigh` per set (lexicographic kept-set order)."""
  D = np.asarray(dist, dtype=np.float64)
  n = D.shape[0]
  m = n - f
  out = []
  for S in itertools.combinations(range(n), m):
    DS = D[np.ix_(S, S)]
    if not np.isfinite(DS).all():
      out.append(np.inf)
      continue
    if m < 2:
      out.append(0.0)
      continue
    r = np.array([_ops._serial_sum(row) for row in DS]) / float(m)
    g = _ops._serial_sum(r) / float(m)
    B = -0.5 * (((DS - r[:, None]) - r[None, :]) + g)
    out.append(float(np.max(_ops.dnc_eigh(B)[0])))
  return np.array(out)


def _psd_case(n, d, seed, scale=1.0):
  gen = torch.Generator().manual_seed(seed)
  G = torch.randn(n, d, generator=gen) * scale
  return G, _ops.torch_pairwise_distances(G)


@pytest.mark.parametrize("n,f,d", [(3, 1, 5), (5, 2, 3), (8, 2, 16), (9, 3, 40), (12, 4, 7), (10, 0, 6), (7, 3, 2)])
def test_scores_equal_per_set_jacobi_bit_for_bit(n, f, d):
  G, D = _psd_case(n, d, seed=n * 31 + f)
  scores = _ops.smea_scores(D, f)
  assert scores.shape == (math.comb(n, f),)
  expect = _per_set_scores(D.numpy(), f)
  assert np.array_equal(scores.view(np.int64), expect.view(np.int64)), (scores, expect)


def _oracle(G, f):
  """float64 lambda_max of the covariance (1/m sum of the centred rows' outer products) of every kept set, lexicographic order."""
  X = G.double().numpy()
  n = X.shape[0]
  out = []
  for S in itertools.combinations(range(n), n - f):
    Y = X[list(S)] - X[list(S)].mean(axis=0)
    out.append(float(np.linalg.eigvalsh(Y.T @ Y / len(S))[-1]) if Y.shape[1] <= Y.shape[0] else float(np.linalg.eigvalsh(Y @ Y.T / len(S))[-1]))
  return np.array(out)


@pytest.mark.parametrize("n,f,d,seed", [(6, 1, 50, 1), (8, 2, 20, 2), (9, 2, 300, 3), (11, 3, 64, 4), (13, 4, 9, 5)])
def test_scores_and_selection_against_the_covariance_oracle(n, f, d, seed):
  G, D = _psd_case(n, d, seed)
  G[n - 1] += 0.7   # one shifted row: the sets without it stand out
  D = _ops.torch_pairwise_distances(G)
  m = n - f
  scores = _ops.smea_scores(D, f)
  lam = _oracle(G, f)
  # each fp32 distance is its float64 value within a relative (d + 2) u (the rows are exact in float64); B_S moves by at most
  # 2 max|dD| per entry, lambda_max(B_S) by at most m times that, and score / m by 2 (d + 2) u max D; the Jacobi adds ~1e-15 relative
  bound = 2 * (d + 2) * U * float(D.max()) + 1e-12 * float(lam.max())
  assert float(np.abs(scores / m - lam).max()) <= bound
  # the oracle's best set is selected wherever its runner-up is farther than twice the bound (relative gap over 2 bound / lambda_best)
  order = np.argsort(lam, kind="stable")
  ids = _ops.smea_select(D, f)
  if lam[order[1]] - lam[order[0]] > 2 * bound:
    assert ids.tolist() == list(list(itertools.combinations(range(n), m))[order[0]])
  else:   # not separated: the selection is still among the near-ties
    chosen = list(itertools.combinations(range(n), m)).index(tuple(ids.tolist()))
    assert lam[chosen] - lam[order[0]] <= 2 * bound


def test_rows_spread_along_one_direction_are_removed():
  n, f, d = 10, 2, 40
  gen = torch.Generator().manual_seed(7)
  G = torch.randn(n, d, generator=gen) * 0.1
  v = torch.randn(d, generator=gen)
  v /= v.norm()
  mu = G[:n - f].mean(dim=0)
  # the two Byzantine rows sit on either side of the honest mean along v, within twice the honest rows' distance to it (about 0.63):
  # together they stretch the covariance along v to 2 / 8 = 0.25, far above what the honest rows spread along any direction
  G[n - 2] = mu + v
  G[n - 1] = mu - v
  assert float((G[n - 1] - mu).norm()) < 2 * float((G[:n - f] - mu).norm(dim=1).max())
  ids = _ops.smea_select(_ops.torch_pairwise_distances(G), f)
  assert ids.tolist() == list(range(n - f))
  _equal_bits(_ops.host_smea(G, f), _ops.selection_mean(G, np.arange(n) < n - f))


def test_f_zero_is_the_mean_of_all_rows():
  G, _ = _psd_case(7, 301, seed=9)
  out, _, ids, _ = _ops.host_smea(G, 0, return_details=True)
  assert ids.tolist() == list(range(7))
  acc = torch.zeros(301)
  for i in range(7):
    acc = acc + G[i]
  _equal_bits(out, acc / 7)
  _equal_bits(_ops.torch_smea(G, 0), out)


def test_non_finite_rows_score_inf_and_are_not_selected():
  n, f = 8, 2
  G, _ = _psd_case(n, 33, seed=11)
  G[2, 5] = float("nan")
  G[6, :] = float("inf")
  D = _ops.torch_pairwise_distances(G)
  scores = _ops.smea_scores(D, f)
  for k, S in enumerate(itertools.combinations(range(n), n - f)):
    assert math.isinf(scores[k]) == (2 in S or 6 in S)
  ids = _ops.smea_select(D, f)
  assert ids.tolist() == [0, 1, 3, 4, 5, 7]
  assert bool(torch.isfinite(_ops.host_smea(G, f)).all())
  # every set holds a non-finite distance: all score +inf, the lexicographically smallest set is kept
  G[0, 0] = float("nan")
  G[1, 0] = float("nan")
  ids, score = _ops.smea_select(_ops.torch_pairwise_distances(G), f, return_score=True)
  assert ids.tolist() == list(range(n - f)) and score == math.inf


def test_exact_ties_go_to_the_lexicographically_smallest_set():
  E = torch.eye(9)   # pairwise equidistant rows: every set has the same B_S, so the same score bits
  scores = _ops.smea_scores(_ops.torch_pairwise_distances(E), 3)
  assert len(set(scores.tolist())) == 1
  assert _ops.smea_select(_ops.torch_pairwise_distances(E), 3).tolist() == list(range(6))
  # integer points on a line: {0, 1, 2} and {1, 2, 3} tie (same spread), {0, 1, 2} wins
  G = torch.tensor([0.0, 1.0, 2.0, 3.0, 40.0]).unsqueeze(1)
  scores = _ops.smea_scores(_ops.torch_pairwise_distances(G), 2)
  sets = list(itertools.combinations(range(5), 3))
  assert scores[sets.index((0, 1, 2))] == scores[sets.index((1, 2, 3))]
  assert _ops.smea_select(_ops.torch_pairwise_distances(G), 2).tolist() == [0, 1, 2]


def test_negative_zero_ties_with_positive_zero(monkeypatch):
  # identical rows: B_S = -1/2 (0 + 0) = -0 everywhere, the score of every set is -0; the selection reports +0
  G = torch.ones(6, 5)
  scores = _ops.smea_scores(_ops.torch_pairwise_distances(G), 2)
  assert all(s == 0 and math.copysign(1.0, s) == -1.0 for s in scores)
  ids, score = _ops.smea_select(_ops.torch_pairwise_distances(G), 2, return_score=True)
  assert ids.tolist() == [0, 1, 2, 3] and math.copysign(1.0, score) == 1.0
  # the keys alone: -0 and +0 tie whatever their order, the lexicographically first set wins; NaN counts as +inf
  D = torch.zeros(4, 4)
  # kept sets in lexicographic order: (0, 1, 2), (0, 1, 3), (0, 2, 3), (1, 2, 3)
  for fake, expect in (([1.0, -0.0, 0.0, 2.0], [0, 1, 3]), ([1.0, 0.0, -0.0, 2.0], [0, 1, 3]), ([math.nan, math.inf, 5.0, 5.0], [0, 2, 3]),
                       ([math.nan, math.inf, math.nan, math.inf], [0, 1, 2])):
    monkeypatch.setattr(_ops, "smea_scores", lambda dist, f, fake=fake: np.array(fake))
    ids, score = _ops.smea_select(D, 1, return_score=True)
    assert ids.tolist() == expect, (fake, ids)
    assert math.copysign(1.0, score) == 1.0


def _layout(d):
  layout = FlatLayout()
  layout.add("theta", (d,))
  layout.freeze()
  return layout


@pytest.mark.parametrize("mix", [None, "nnm", "arc", "arc+nnm"])
def test_host_engine_matches_the_torch_reference(mix):
  n, f, d = 9, 2, 1003
  gar = aggregators.instantiate("smea", n, f, [])
  layout = _layout(d)
  engine = HostAggregation(gar, layout, n, build(optimizers, "optimizer", "sgd", []), pre_aggregation=mix, nb_decl_byz=f)
  for step in range(2):
    gen = torch.Generator().manual_seed(13 * step + 1)
    G = torch.zeros(n, layout.padded_size)
    # a tight honest cluster away from the origin and two large rows pointing elsewhere: after ARC clips them they still stand apart,
    # so no two kept sets score close enough for the host's and torch's fp32 distances to order them differently
    G[:, :d] = 3.0 + 0.1 * torch.randn(n, d, generator=gen)
    G[n - 1, :d] = G[n - 1, :d] * -30
    G[n - 2, :d] = G[n - 2, :d] * torch.randn(d, generator=gen).sign() * 20
    engine.grads.copy_(G)
    engine.step(0.1)
    _equal_bits(engine.last_aggregate, _ops.torch_smea(_ops.torch_pre_aggregate(G, mix, f, host=True), f))


def test_argument_errors():
  with pytest.raises(tools.UserException, match="2 f < n"):
    aggregators.instantiate("smea", 8, 4, [])
  with pytest.raises(tools.UserException, match="2 f < n"):
    _ops.check_smea(5, -1)
  with pytest.raises(tools.UserException, match="2\\^14"):
    aggregators.instantiate("smea", 32, 4, [])   # C(32, 4) = 35960
  with pytest.raises(tools.UserException, match="2\\^14"):
    _ops.smea_scores(torch.zeros(20, 20), 6)   # C(20, 6) = 38760
  for n, f in ((16, 7), (20, 5), (26, 4), (32, 3)):   # the largest f of each n
    _ops.check_smea(n, f)
    with pytest.raises(tools.UserException, match="2\\^14"):
      _ops.check_smea(n + 1, f + 1)
  with pytest.raises(tools.UserException, match="no --aggregator-args"):
    aggregators.instantiate("smea", 8, 2, ["iterations:3"])
  assert aggregators.instantiate("smea", 8, 2, None).fused_spec().rule == "smea"


def test_rule_id():
  assert FusedSpec.RULES.index("smea") == 11
  assert FusedSpec.RULES[:11] == ("average", "average-nan", "median", "averaged-median", "krum", "bulyan", "trimmed-mean", "mda",
                                  "geometric-median", "centered-clipping", "dnc")
  assert "smea" in FusedSpec.RULES_WITH_F
  spec = FusedSpec("smea", 8, f=2)
  assert spec.rule_id == 11 and spec.with_mix("nnm").rule == "smea"


def test_mnist_under_alie_loss_decreases():
  n, f, steps = 7, 2, 8
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate("smea", n, f, [])
  attack = attacks.instantiate("alie", n, f, [])
  mgr = Manager(experiment, gar, n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu", attack=attack, nb_real_byz=f, seed=1)
  losses = [float(mgr.train()) for _ in range(steps)]
  assert all(math.isfinite(v) for v in losses)
  assert losses[-1] < losses[0], losses

"""Trimmed mean and MDA (minimum-diameter averaging) on the host: the C++ library against the float64 torch oracle, exact cases
on small-integer data, the MDA tie-break, non-finite inputs, invariances, argument checks and CPU training runs."""

import itertools
import math

import pytest
import torch

from aggregathor_b200 import aggregators, attacks, experiments, tools
from aggregathor_b200.aggregators import FusedSpec, _ops
from aggregathor_b200.engine.trainer import Manager

DTYPES = [torch.float32, torch.float64]


def _data(n, d, seed, outliers=0, dtype=torch.float32):
  gen = torch.Generator().manual_seed(seed)
  G = torch.randn(n, d, generator=gen, dtype=torch.float64)
  for k in range(outliers):
    G[n - 1 - k] = G[n - 1 - k] * 25 - 4
  return G.to(dtype)


def _integers(n, d, seed, low=-8, high=9):
  gen = torch.Generator().manual_seed(seed)
  return torch.randint(low, high, (n, d), generator=gen).float()


def _close(a, b, tol):
  a, b = a.double(), b.double()
  assert bool((torch.isnan(a) == torch.isnan(b)).all())
  a, b = torch.nan_to_num(a), torch.nan_to_num(b)
  assert float((a - b).abs().max()) <= tol * max(1.0, float(b.abs().max())), float((a - b).abs().max())


def _tm_cases():
  for n in (3, 5, 8, 11, 19, 33, 40):
    for f in sorted({0, 1, n // 4, (n - 1) // 2}):
      yield n, f


def _mda_cases():
  for n in (3, 5, 8, 11, 19, 33, 40):
    for f in sorted({0, 1, min(3, (n - 1) // 2), (n - 1) // 2 if n <= 19 else 3}):
      yield n, f


def test_rule_ids_are_appended():
  assert FusedSpec.RULES[:6] == ("average", "average-nan", "median", "averaged-median", "krum", "bulyan")
  assert FusedSpec("trimmed-mean", 8, f=2).rule_id == 6 and FusedSpec("mda", 8, f=2).rule_id == 7


def test_registered():
  names = set(aggregators.itemize())
  assert {"trimmed-mean", "mda"} <= names
  assert aggregators.instantiate("trimmed-mean", 7, 2, []).fused_spec().rule == "trimmed-mean"
  spec = aggregators.instantiate("mda", 7, 2, []).fused_spec()
  assert (spec.rule, spec.n, spec.f) == ("mda", 7, 2)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n,f", list(_tm_cases()))
def test_trimmed_mean_host_matches_float64_oracle(n, f, dtype):
  G = _data(n, 1001, seed=n * 31 + f, outliers=f, dtype=dtype)
  out = _ops.host_trimmed_mean(G, f)
  assert out.dtype == dtype
  _close(out, _ops.torch_trimmed_mean(G.double(), f), 2e-6 if dtype == torch.float32 else 1e-13)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n,f", list(_mda_cases()))
def test_mda_host_matches_float64_oracle(n, f, dtype):
  G = _data(n, 517, seed=n * 17 + f, outliers=f, dtype=dtype)
  out, selected = _ops.host_mda(G, f, return_selected=True)
  assert out.dtype == dtype and selected.tolist() == sorted(selected.tolist()) and len(selected) == n - f
  # the selection is a function of the distance matrix: check it on the host's own distances, whatever their rounding
  dist = _ops.host_pairwise_distances(G)
  assert torch.equal(_ops.mda_select(dist.double(), f), selected)
  assert torch.equal(_ops.host_mda_select(dist, f), selected)
  _close(out, G.double()[selected].sum(dim=0) / (n - f), 2e-6 if dtype == torch.float32 else 1e-13)
  if dtype == torch.float64:
    ref, ref_selected = _ops.torch_mda(G, f, return_selected=True)
    assert torch.equal(ref_selected, selected)
    _close(out, ref, 1e-13)
  if f:   # the outliers are the last f rows
    assert selected.tolist() == list(range(n - f))


@pytest.mark.parametrize("n,f", [(3, 1), (5, 2), (8, 2), (11, 3), (19, 4), (33, 5), (40, 2)])
def test_exact_on_small_integers(n, f):
  """Every sum of small integers is exact, so the fp32 host results must equal the float64 oracle rounded once, bit for bit
  (a quotient of two fp32 values computed in float64 then rounded to fp32 is correctly rounded). Integer data also has many
  tied values and tied distances: both back-ends must break them the same way."""
  G = _integers(n, 257, seed=n + 100 * f)
  assert torch.equal(_ops.host_trimmed_mean(G, f), _ops.torch_trimmed_mean(G.double(), f).float())
  assert torch.equal(_ops.host_trimmed_mean(G.double(), f), _ops.torch_trimmed_mean(G.double(), f))
  fm = min(f, 3)
  out, selected = _ops.host_mda(G, fm, return_selected=True)
  ref, ref_selected = _ops.torch_mda(G.double(), fm, return_selected=True)
  assert torch.equal(selected, ref_selected)
  assert torch.equal(out, ref.float())


def test_trimmed_mean_f0_is_the_plain_mean():
  G = _integers(9, 301, seed=4)
  assert torch.equal(_ops.host_trimmed_mean(G, 0), _ops.host_average(G))
  G[2, 5] = float("nan")
  out = _ops.host_trimmed_mean(G, 0)
  assert bool(torch.isnan(out[5])) and int(torch.isnan(out).sum()) == 1


@pytest.mark.parametrize("dist_of,f,expected", [
  # four points on a line, 0 1 2 3: {0,1,2} and {1,2,3} both have diameter 4
  ([0.0, 1.0, 2.0, 3.0], 1, [0, 1, 2]),
  # 5 10 0 10 0 ... two tied pairs of clusters: {0,1,3} and {0,2,4} have diameter 25; the lexicographically smaller wins
  ([5.0, 0.0, 10.0, 0.0, 10.0], 2, [0, 1, 3]),
  ([10.0, 0.0, 10.0, 0.0, 5.0], 2, [0, 2, 4]),
  ([0.0, 10.0, 5.0, 10.0, 0.0], 2, [0, 2, 4]),
])
def test_mda_tie_break_on_a_line(dist_of, f, expected):
  G = torch.tensor(dist_of).unsqueeze(1)
  for dtype in DTYPES:
    Gd = G.to(dtype)
    _, selected = _ops.host_mda(Gd, f, return_selected=True)
    assert selected.tolist() == expected
    assert _ops.torch_mda(Gd, f, return_selected=True)[1].tolist() == expected


@pytest.mark.parametrize("n,f", [(4, 1), (7, 3), (12, 2)])
def test_mda_tie_break_equidistant(n, f):
  """The rows of the identity are pairwise equidistant: every subset ties, the first n - f workers win."""
  G = torch.eye(n)
  assert _ops.host_mda(G, f, return_selected=True)[1].tolist() == list(range(n - f))
  # two equidistant clusters far apart: the larger one holds n - f members only if it is picked whole
  D = torch.ones(n, n) - torch.eye(n)
  D[:, n - 1] = D[n - 1, :] = 100.0
  D[n - 1, n - 1] = 0.0
  assert _ops.host_mda_select(D, f).tolist() == list(range(n - f))
  assert _ops.mda_select(D.double(), f).tolist() == list(range(n - f))


def test_mda_select_tie_key_against_brute_force():
  """Quantised random distance matrices (many ties) vs a direct transcription of the rule over every kept set."""
  gen = torch.Generator().manual_seed(3)
  for trial in range(20):
    n = 5 + trial % 6
    f = trial % ((n - 1) // 2 + 1)
    D = torch.randint(0, 4, (n, n), generator=gen).double()
    D = torch.triu(D, 1)
    D = D + D.T
    if trial % 3 == 0:
      D[0, 1] = D[1, 0] = float("nan")
    key = lambda S: (max([float(D[i, j]) if D[i, j] == D[i, j] else math.inf for i, j in itertools.combinations(S, 2)] or [0.0]), S)
    expected = min(itertools.combinations(range(n), n - f), key=key)
    assert _ops.host_mda_select(D, f).tolist() == list(expected), (n, f)
    assert _ops.host_mda_select(D.float(), f).tolist() == list(expected), (n, f)
    assert _ops.mda_select(D, f).tolist() == list(expected), (n, f)


def test_trimmed_mean_drops_up_to_f_non_finite_values():
  n, f, d = 9, 3, 2000
  G = _data(n, d, seed=12)
  gen = torch.Generator().manual_seed(13)
  bad = [float("nan"), float("inf"), float("-inf")]
  for x in range(d):
    count = int(torch.randint(0, f + 1, (1,), generator=gen))
    rows = torch.randperm(n, generator=gen)[:count]
    for k, row in enumerate(rows.tolist()):
      G[row, x] = bad[(x + k) % 3]
  for dtype in DTYPES:
    out = _ops.host_trimmed_mean(G.to(dtype), f)
    assert bool(torch.isfinite(out).all())
    _close(out, _ops.torch_trimmed_mean(G.double(), f), 2e-6 if dtype == torch.float32 else 1e-13)
  # more than f non-finite values: one of them is kept
  G[:f + 1, 0] = float("nan")
  assert bool(torch.isnan(_ops.host_trimmed_mean(G, f)[0]))


def test_mda_excludes_a_nan_row():
  for n, f in ((5, 1), (8, 2), (11, 3)):
    G = _data(n, 300, seed=n)
    G[2, 17] = float("nan")
    for dtype in DTYPES:
      out, selected = _ops.host_mda(G.to(dtype), f, return_selected=True)
      assert 2 not in selected.tolist() and bool(torch.isfinite(out).all())
      assert 2 not in _ops.torch_mda(G.to(dtype), f, return_selected=True)[1].tolist()


def test_invariances():
  n, f = 9, 2
  G = _integers(n, 400, seed=8)
  perm = torch.randperm(n, generator=torch.Generator().manual_seed(1))
  shift = _integers(1, 400, seed=9)
  # trimmed mean: exact on integers whatever the row order; shifts with the data (up to the rounding of the final division)
  assert torch.equal(_ops.host_trimmed_mean(G[perm], f), _ops.host_trimmed_mean(G, f))
  _close(_ops.host_trimmed_mean(G + shift, f), _ops.host_trimmed_mean(G, f) + shift[0], 1e-6)
  # MDA: translation leaves every distance unchanged, hence the selection; the permuted rows select the permuted set
  out, selected = _ops.host_mda(G, f, return_selected=True)
  out_t, selected_t = _ops.host_mda(G + shift, f, return_selected=True)
  assert torch.equal(selected_t, selected)
  _close(out_t, out + shift[0], 1e-6)
  R = _data(n, 400, seed=10, outliers=f)
  out, selected = _ops.host_mda(R, f, return_selected=True)
  out_p, selected_p = _ops.host_mda(R[perm], f, return_selected=True)
  assert sorted(perm[selected_p].tolist()) == selected.tolist()
  _close(out_p, out, 1e-6)


def test_argument_checks():
  for name in ("trimmed-mean", "mda"):
    with pytest.raises(tools.UserException):
      aggregators.instantiate(name, 6, 3, [])
    with pytest.raises(tools.UserException):
      aggregators.instantiate(name, 4, 2, [])
    aggregators.instantiate(name, 7, 3, [])
  with pytest.raises(tools.UserException):
    aggregators.instantiate("mda", 32, 7, [])           # C(32, 7) = 3365856 > 2^20
  aggregators.instantiate("mda", 32, 6, [])             # C(32, 6) = 906192
  aggregators.instantiate("mda", 19, 9, [])
  G = _data(6, 10, seed=0)
  with pytest.raises(tools.UserException):
    _ops.host_trimmed_mean(G, 3)
  with pytest.raises(tools.UserException):
    _ops.torch_trimmed_mean(G, 3)
  with pytest.raises(tools.UserException):
    _ops.host_mda(G, 3)
  with pytest.raises(tools.UserException):
    _ops.torch_mda(G, 3)
  with pytest.raises(tools.UserException):
    _ops.host_mda_select(torch.zeros(32, 32), 7)
  # the C++ library checks the bound by itself too
  import ctypes
  D = torch.zeros(32, 32)
  sel = torch.zeros(32, dtype=torch.int64)
  assert _ops._host("mda_select", torch.float32)(_ops._ptr(D), ctypes.c_size_t(32), ctypes.c_size_t(7), _ops._ptr(sel)) != 0
  assert _ops._host("mda_select", torch.float32)(_ops._ptr(D), ctypes.c_size_t(32), ctypes.c_size_t(6), _ops._ptr(sel)) == 0
  # a plug-in built for more workers than it is given re-checks with the actual n
  with pytest.raises(tools.UserException):
    aggregators.instantiate("trimmed-mean", 9, 3, []).aggregate(list(_data(6, 10, seed=1)))


def _manager(gar_name, n, f, attack=None, real=0):
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate(gar_name, n, f, [])
  return Manager(experiment, gar, n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu", attack=attack, nb_real_byz=real)


@pytest.mark.parametrize("rule", ["trimmed-mean", "mda"])
def test_training_under_flip_attack(rule):
  mgr = _manager(rule, 7, 2, attacks.instantiate("flip", 7, 2, ["factor:-50"]), 2)
  first = float(mgr.train())
  for _ in range(25):
    last = float(mgr.train())
  assert last == last and last < first
  assert mgr.evaluate()["top1-X-acc"] > 0.5

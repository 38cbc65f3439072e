"""The six original aggregation rules of the fused sm_90a kernel (`native/op_gar/gar.cu`: average, average-nan, median,
averaged-median, Krum and Bulyan) against float64 oracles.

Every oracle below is plain NumPy float64 code that spells out the rule it asserts; it does not call `_ops` or the host library
`gars.cpp`. `test_oracles_*` check the oracles themselves without a GPU: against the original AggregaThor's stored outputs, against the
host and torch rules on tie-free data, and on small hand-computed cases.

The ordering convention of every rule (`before()` in `agb_device.cuh`): finite values ascending, then the non-finite values (NaN, +Inf
and -Inf alike), ties to the lower index; -0 and +0 compare equal.

Operands come in two families:
  * grid operands: small integers, with the range chosen so that every squared distance and every Krum / Bulyan score is at most
    2^24. Every fp32 partial sum is then exact whatever the fold order or FMA contraction, and the only roundings left are the ones
    the rule defines (one division, one fp32 deviation), which the oracle performs once too. Outputs, the [n, n] distance matrix,
    the selection masks and theta are asserted bit for bit; Bulyan's final beta-average (of non-integer theta means) within a bound;
  * random operands with Byzantine rows (scaled x30, shifted, partly non-finite): distances within a per-pair bound, outputs within
    bounds derived next to each assert, and masks exactly, after the case has asserted that its selection margins exceed the bounds.

Every GPU case counts the calls that reached `FusedLauncher.launch` (and replaces the torch fall-back with a failure), so it proves
the sm_90a kernel served it.
"""

import math
import pathlib

import numpy as np
import pytest
import torch

from aggregathor_b200.aggregators import FusedSpec, _ops

gpu = pytest.mark.gpu
U = 2.0 ** -24                         # unit roundoff of fp32 (round to nearest)
GOLDEN = pathlib.Path(__file__).resolve().parent / "golden" / "reference_native_gars.npz"
SENTINEL = 0x7fc0beef                  # a quiet NaN with a payload: agg_out outside the owned segments must keep these bits
COORD_RULES = ("average", "average-nan", "median", "averaged-median")
COORD_N = (1, 2, 3, 7, 8, 9, 15, 16, 17, 24, 31, 32)


def gamma(k):
  """gamma_k = k u / (1 - k u): the relative error bound of k fp32 roundings in sequence (Higham, Lemma 3.1)."""
  return k * U / (1 - k * U)


# ---------------------------------------------------------------------------- #
# float64 oracles

def order_key(values):
  """The order key: a finite value is itself, a non-finite value (NaN, +Inf, -Inf) is +inf, after every finite value. A stable sort
  on it puts ties (-0 and +0 included, since they compare equal) in index order."""
  values = np.asarray(values, dtype=np.float64)
  return np.where(np.isfinite(values), values, np.inf)


def ranks(V):
  """The rank of every entry of V along axis 0 under the order key: the number of entries ordered before it."""
  order = np.argsort(order_key(V), axis=0, kind="stable")
  out = np.empty_like(order)
  np.put_along_axis(out, order, np.arange(V.shape[0]).reshape((-1,) + (1,) * (V.ndim - 1)), axis=0)
  return out


def serial_sum(X, keep=None):
  """The sum over the rows of X (float64) in index order, from +0; with `keep` (bool, X's shape) only the kept entries."""
  s = np.zeros(X.shape[1:], dtype=np.float64)
  with np.errstate(invalid="ignore"):
    for i in range(X.shape[0]):
      s = s + (X[i] if keep is None else np.where(keep[i], X[i], 0.0))
  return s


def rounded(num, den):
  """fp32(num / den), rounded once. On grid operands num is an exact integer (|num| < 2^24) and den <= 32: if the float64 quotient
  landed on an fp32 midpoint M = k 2^e (k < 2^25) without being exact, |num - den M| would be a nonzero multiple of min(1, 2^e) below
  den M 2^-53 < 2^(e - 23) (e < 0) or below 1 (e >= 0), which is impossible; so going through float64 cannot double-round. On random
  operands the fp32 quotient is the reference the kernel's result is bounded against."""
  with np.errstate(invalid="ignore", divide="ignore"):
    return (np.asarray(num, dtype=np.float64) / den).astype(np.float32)


def average_ref(X):
  """average: the sum over i added from +0, divided once by n (a column of -0 gives +0)."""
  return rounded(serial_sum(X), X.shape[0])


def average_nan_ref(X):
  """average-nan: the sum of the finite values added from +0, divided once by their count; no finite value gives 0 / 0 = NaN."""
  finite = np.isfinite(X)
  return rounded(serial_sum(X, finite), finite.sum(axis=0))


def median_ref(X):
  """median: the value ranked n // 2 (the upper median), returned with its own bits (a -0 / +0 tie returns the lower index's zero)."""
  n = X.shape[0]
  return np.take_along_axis(X, np.argsort(order_key(X), axis=0, kind="stable")[n // 2][None], axis=0)[0].astype(np.float32)


def deviations(X, med):
  """d_i = fp32(|v_i - median|). The float64 difference of two fp32 values is exact unless their exponents differ by more than 29, and
  then the fp32 rounding gives the larger operand's magnitude either way, so the one fp32 rounding here is the kernel's."""
  with np.errstate(invalid="ignore"):
    return np.abs(X - med.astype(np.float64)).astype(np.float32)


def averaged_median_ref(X, beta, exact=False):
  """averaged-median(beta): the beta values with the smallest deviation d_i = fp32(|v_i - median|), ranked under the order key (two
  deviations that differ exactly may round to the same fp32 value and then tie by index), summed in index order from +0 and divided
  once by beta. -> (fp32 result, the float64 sum, the [n, d] selection). `exact`: the float64 quotient instead (random operands)."""
  keep = ranks(deviations(X, median_ref(X))) < beta
  total = serial_sum(X, keep)
  return (total / beta if exact else rounded(total, beta)), total, keep


def distances_ref(X):
  """D_ij = sum (x_i - x_j)^2 in float64, any non-finite value replaced by +inf; the diagonal is 0."""
  n = X.shape[0]
  D = np.zeros((n, n))
  with np.errstate(invalid="ignore", over="ignore"):
    for i in range(n):
      D[i] = ((X - X[i]) ** 2).sum(axis=1)
  D[~np.isfinite(D)] = np.inf
  np.fill_diagonal(D, 0.0)
  return D


def _item_key(value, index):
  """The order key of one value with its index, for Python sorts: finite values ascending, non-finite last, ties -> lower index."""
  return (0, value, index) if math.isfinite(value) else (1, 0.0, index)


def neighbours(D, k):
  """For every row i: the rows j != i in order (D_ij under the order key, ties -> lower j); the first k are i's scored neighbours."""
  n = D.shape[0]
  return [sorted((j for j in range(n) if j != i), key=lambda j: _item_key(float(D[i, j]), j)) for i in range(n)]


def krum_ref(X, f, m, D=None):
  """Krum(f, m): score_i is the sum of the n - f - 2 smallest D_ij (j != i), added in ascending order; the m lowest scores are
  selected, index-stable (non-finite scores last); the output is the mean of the selected rows, added in worker order from +0 and
  divided once by m. -> (fp32 output, selection mask, scores, D)."""
  n = X.shape[0]
  D = distances_ref(X) if D is None else D
  k = n - f - 2
  scores = [sum(float(D[i, j]) for j in near[:k]) for i, near in enumerate(neighbours(D, k))]
  chosen = sorted(range(n), key=lambda i: _item_key(scores[i], i))[:m]
  mask = sum(1 << i for i in chosen)
  keep = np.array([(mask >> i) & 1 for i in range(n)], dtype=bool)
  return rounded(serial_sum(X, np.broadcast_to(keep[:, None], X.shape)), m), mask, scores, D


def bulyan_ref(X, f, m, D=None):
  """Bulyan(f, m) (DESIGN.md, section 2, steps 4 and 5): theta = n - 2f - 2 rounds on the distances D. Row i's score is the sum of its
  k = n - f - 2 nearest D_ij (ascending); its f + 1 farthest neighbours are pruned (never counted, so never subtracted). Round r ranks
  the rows not yet removed first, each group by score under the order key, selects the first m - r, and removes the first one (the
  best); every row still present subtracts its distance to the best if the best is one of its k scored neighbours, 0 otherwise. Each
  round's mean is the sum of its selected rows in worker order from +0, divided once by m - r (rounded to fp32); the output is the
  averaged median of the theta means with beta = theta - 2f. -> (output, masks, fp32 theta means [theta, d], D, whether some round's
  best row was a pruned neighbour of a row still present, the float64 sum of the output and the beta-selection of the means)."""
  n = X.shape[0]
  D = distances_ref(X) if D is None else D
  theta, k = n - 2 * f - 2, n - f - 2
  near = neighbours(D, k)
  scores = [sum(float(D[i, j]) for j in near[i][:k]) for i in range(n)]
  scored = [set(near[i][:k]) for i in range(n)]
  removed = [False] * n
  masks, means, pruned_best = [], [], False
  for r in range(theta):
    order = sorted(range(n), key=lambda i: (removed[i],) + _item_key(scores[i], i))
    chosen = order[:m - r]
    masks.append(sum(1 << i for i in chosen))
    keep = np.zeros(X.shape, dtype=bool)
    keep[chosen] = True
    means.append(rounded(serial_sum(X, keep), m - r))
    best = order[0]
    removed[best] = True
    for i in range(n):
      if not removed[i]:
        if best in scored[i]:
          scores[i] -= float(D[i, best])
        elif D[i, best] > 0:
          pruned_best = True
  means = np.stack(means)
  out, total, keep = averaged_median_ref(means.astype(np.float64), theta - 2 * f)
  return out, masks, means, D, pruned_best, total, keep


# ---------------------------------------------------------------------------- #
# Operands

def grid_rows(n, d, seed, R):
  """[n, d] small integers in [-R, R] (many ties), fp32."""
  return np.random.default_rng(seed).integers(-R, R + 1, size=(n, d)).astype(np.float32)


def special_columns(n, rng):
  """Edge columns of n values: -0 only, +-0 ties at the median, median +- k pairs, single NaN / +Inf / -Inf, more than n / 2
  non-finite values, none finite, and +Inf with -Inf."""
  nz = np.float32(-0.0)
  signs = np.array([nz if i % 2 else np.float32(0.0) for i in range(n)], dtype=np.float32)
  pairs = [1.0] + [v for k in range(1, n) for v in (1.0 + k, 1.0 - k)]
  cols = [np.full(n, nz, dtype=np.float32), signs, -signs, rng.permutation(np.array(pairs[:n], dtype=np.float32))]
  for special in (np.nan, np.inf, -np.inf):
    col = rng.integers(-2, 3, size=n).astype(np.float32)
    col[rng.integers(n)] = special
    cols.append(col)
  many = rng.integers(-2, 3, size=n).astype(np.float32)
  many[rng.permutation(n)[:n // 2 + 1]] = rng.choice(np.array([np.nan, np.inf, -np.inf], dtype=np.float32), size=n // 2 + 1)
  cols.append(many)
  cols.append(rng.choice(np.array([np.nan, np.inf, -np.inf], dtype=np.float32), size=n))
  both = rng.integers(-2, 3, size=n).astype(np.float32)
  both[:min(n, 2)] = (np.inf, -np.inf)[:min(n, 2)]
  cols.append(both)
  return cols


def coordinate_operands(n, d, seed, bad_rows=False):
  """Grid operands with ties for the coordinate rules: integers in [-3, 3], the special columns at random positions (as many as fit),
  and with `bad_rows` a whole NaN row and a whole -Inf row."""
  rng = np.random.default_rng(seed)
  X = grid_rows(n, d, seed, 3)
  cols = special_columns(n, rng)
  for col, x in zip(cols, rng.permutation(d)):
    X[:, x] = col
  if bad_rows and n >= 3:
    X[rng.integers(n)] = np.nan
    X[rng.integers(n)] = -np.inf
  return X


def distance_range(n, f, d):
  """The largest R with every score at most 2^24: a score adds n - f - 2 distances of at most d (2R)^2."""
  R = min(8, int(math.isqrt((1 << 24) // (4 * d * max(1, n - f - 2)))))
  assert R >= 1
  return R


def distance_operands(n, f, d, seed, bad=False):
  """Grid operands for Krum and Bulyan: integers in [-R, R], R from `distance_range`; a few duplicated rows (equal distances, equal
  scores), the last f rows shifted to +R (Byzantine). `bad`: a +Inf row and a row with NaN spots, whose distances are +inf."""
  R = distance_range(n, f, d)
  rng = np.random.default_rng(seed)
  X = grid_rows(n, d, seed, R)
  for _ in range(n // 4):
    i, j = rng.choice(n, size=2, replace=False)
    X[j] = X[i]
  for k in range(f):
    X[n - 1 - k] = np.clip(X[n - 1 - k] + R, -R, R)
  if bad:
    X[1] = np.inf
    X[n - 2, ::3] = np.nan
  return X


def random_operands(n, d, seed, byzantine=()):
  """randn rows; Byzantine rows (listed by kind) from the last row down: "scaled" x30, "shifted" +5, "spotted" NaN and +-Inf spots."""
  rng = np.random.default_rng(seed)
  X = rng.standard_normal((n, d)).astype(np.float32)
  for k, kind in enumerate(byzantine):
    row = n - 1 - k
    if kind == "scaled":
      X[row] *= 30
    elif kind == "shifted":
      X[row] += 5
    else:
      X[row, 1::7] = np.nan
      X[row, 4::11] = np.inf
      X[row, 6::13] = -np.inf
  return X


def threads_vec(n):
  """The coordinates one sweep of one CTA covers in the kernel instance serving n rows (`launch<8, 4>`, `<16, 4>`, `<32, 1>`)."""
  return 512 * 4 if n <= 8 else 256 * 4 if n <= 16 else 256


# ---------------------------------------------------------------------------- #
# Comparisons

def assert_bits(got, want, what=""):
  """fp32 equality bit for bit; NaN positions must match (their payloads may not)."""
  got, want = np.asarray(got, dtype=np.float32), np.asarray(want, dtype=np.float32)
  assert got.shape == want.shape, (what, got.shape, want.shape)
  nan = np.isnan(want)
  assert np.array_equal(np.isnan(got), nan), (what, np.flatnonzero(np.isnan(got) != nan)[:8])
  bad = np.flatnonzero((got.view(np.int32) != want.view(np.int32)) & ~nan)
  assert bad.size == 0, (what, int(bad[0]), float(got.flat[bad[0]]), float(want.flat[bad[0]]))


def assert_within(got, want, bound, what=""):
  """|got - want| <= bound wherever want is finite; identical non-finite values elsewhere (NaN positions, signed infinities)."""
  got = np.asarray(got, dtype=np.float64)
  finite = np.isfinite(want)
  assert np.array_equal(np.isnan(got), np.isnan(want)), (what, np.flatnonzero(np.isnan(got) != np.isnan(want))[:8])
  assert np.array_equal(got[~finite & ~np.isnan(want)], want[~finite & ~np.isnan(want)]), what
  err = np.abs(got[finite] - want[finite])
  over = np.flatnonzero(err > np.broadcast_to(bound, want.shape)[finite])
  assert over.size == 0, (what, int(over[0]), float(err[over[0]]), float(np.broadcast_to(bound, want.shape)[finite][over[0]]))


def assert_distances(dist, D, bound=None):
  """The kernel's [n, n] matrix off the diagonal (never written): bit for bit (grid operands), or within `bound` x D (random ones)."""
  off = ~np.eye(D.shape[0], dtype=bool)
  if bound is None:
    assert_bits(dist[off], D[off].astype(np.float32), "distances")
  else:
    assert_within(dist[off], D[off], bound * np.where(np.isfinite(D[off]), D[off], 0.0), "distances")


def sum_bound(X, keep, count):
  """|fp32(sum) / count - exact| for the kept entries added in fp32 then divided once: gamma_count sum |x| / count (the sum's count - 1
  roundings and the division's one)."""
  count = np.maximum(count, 1)
  return gamma(count) * serial_sum(np.abs(np.where(np.isfinite(X), X, 0.0)), keep) / count


# ---------------------------------------------------------------------------- #
# Kernel runners

@pytest.fixture
def launches(monkeypatch):
  """The list of rules served by `FusedLauncher.launch` during the test; the torch fall-back fails the test."""
  from aggregathor_b200.ops import gar as gar_ops
  served, launch = [], gar_ops.FusedLauncher.launch

  def counted(self, spec, rows, *args, **kwargs):
    served.append(spec.rule)
    return launch(self, spec, rows, *args, **kwargs)

  def no_fall_back(*args, **kwargs):
    raise AssertionError("the torch fall-back served an sm_90a case")

  monkeypatch.setattr(gar_ops.FusedLauncher, "launch", counted)
  monkeypatch.setattr(gar_ops, "_torch_rules", no_fall_back)
  return served


def spec_of(rule, n, f=0, m=0, beta=0):
  if rule == "bulyan":
    beta = n - 4 * f - 2
  return FusedSpec(rule, n, f=f, m=m, beta=beta)


def aggregate(spec, X, offset=False):
  """`ops.gar.aggregate` on X (any d; `offset`: a view 4 bytes into its allocation, so the rows take the `_padded` copy)
  -> (out, dist [n, n], info) as NumPy arrays."""
  from aggregathor_b200.ops import gar as gar_ops
  n, d = X.shape
  G = torch.from_numpy(X).cuda()
  if offset:
    base = torch.empty(n * d + 1, device="cuda")
    base[1:].copy_(G.view(-1))
    G = base[1:].view(n, d)
    assert G.data_ptr() % 16 == 4
  out, dist, info = gar_ops.aggregate(spec, G, return_details=True)[:3]
  return out.cpu().numpy(), dist.cpu().numpy(), info.cpu().numpy()


# launchers of this module alone: `launch` fills their distances and masks with sentinels, and the diagonal of the distance matrix is
# never written, so the cached launchers of `ops.gar.aggregate`, whose callers read that diagonal as +0, must not be touched
_own_launchers = {}


def launch(spec, X, segments=None, staging=False, max_ctas=0, first_seg=0):
  """`FusedLauncher.launch` on X (d % 4 == 0) over the owned `segments` (default: all of [0, d)), agg_out pre-filled with SENTINEL,
  the first `first_seg` segments pre-accumulated by `phase_a`, with or without a staging tile, on at most `max_ctas` CTAs (0: the
  full grid) -> (out [d] with the sentinel outside the segments, dist [n, n], info) as NumPy arrays."""
  from aggregathor_b200.ops import gar as gar_ops
  n, d = X.shape
  segments = [(0, d)] if segments is None else segments
  G = torch.from_numpy(X).cuda()
  rows = [G.data_ptr() + i * d * 4 for i in range(n)]
  out = torch.full((d,), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
  owned = sum(hi - lo for lo, hi in segments)
  tile = torch.full((n, max(owned, 4)), float("nan"), device="cuda") if staging else None
  launcher = _own_launchers.get(n)
  if launcher is None:
    launcher = _own_launchers[n] = gar_ops.FusedLauncher(G.device, n)
  launcher.dist_out.fill_(float("nan"))
  launcher.info.fill_(-7)
  for seg in range(first_seg):
    launcher.phase_a(spec, rows, segments, seg, agg_out=out, staging=tile, first_seg=seg + 1)
  launcher.launch(spec, rows, segments=segments, agg_out=out, staging=tile, first_seg=first_seg, max_ctas_limit=max_ctas)
  return out.cpu().numpy(), launcher.dist_out.view(n, n).cpu().numpy(), launcher.info.cpu().numpy()


def owned_columns(d, segments):
  cols = np.zeros(d, dtype=bool)
  for lo, hi in segments:
    cols[lo:hi] = True
  return cols


def assert_sentinel(out, segments):
  outside = ~owned_columns(out.shape[0], segments)
  assert (out.view(np.int32)[outside] == SENTINEL).all(), np.flatnonzero(out.view(np.int32)[outside] != SENTINEL)[:8]


def masks_of(info, count):
  return [int(info[1 + k]) & 0xffffffff for k in range(count)]


def reference(rule, X, f=0, m=0, beta=0):
  """The oracle's (fp32 output, masks or None, D or None) of one rule on X."""
  if rule == "average":
    return average_ref(X), None, None
  if rule == "average-nan":
    return average_nan_ref(X), None, None
  if rule == "median":
    return median_ref(X), None, None
  if rule == "averaged-median":
    return averaged_median_ref(X, beta)[0], None, None
  if rule == "krum":
    out, mask, _, D = krum_ref(X, f, m)
    return out, [mask], D
  out, masks, _, D, _, _, _ = bulyan_ref(X, f, m)
  return out, masks, D


# ---------------------------------------------------------------------------- #
# CPU self-checks of the oracles

def _golden():
  with np.load(GOLDEN) as data:
    return {key: np.array(data[key]) for key in data.files}


@pytest.mark.parametrize("n,d", [(4, 50), (7, 1001), (8, 4096), (11, 333)])
def test_oracles_reproduce_the_reference_outputs(n, d):
  """The original AggregaThor's median, average-nan and averaged-median (`oracle/make_gars_golden.py`) agree with the oracles. Its
  median is an nth_element under the same key, so it is the same value; its average-nan adds in index order and its averaged-median
  in nth_element's order, both in fp32, so each is within gamma_k sum |x| / k of the exact float64 quotient (k: the count)."""
  g = _golden()
  key = "%d_%d_" % (n, d)
  X, clean = g[key + "G"].astype(np.float64), g[key + "clean"].astype(np.float64)
  assert_bits(g[key + "median"], median_ref(X), "median")
  finite = np.isfinite(X)
  count = finite.sum(axis=0)
  assert_within(g[key + "average_nan"], serial_sum(X, finite) / count, sum_bound(X, finite, count), "average-nan")
  _, total, keep = averaged_median_ref(clean, n - 2)
  assert_within(g[key + "averaged_median"], total / (n - 2), sum_bound(clean, keep, n - 2), "averaged-median")


@pytest.mark.parametrize("n,f,d", [(7, 1, 300), (8, 1, 1000), (11, 2, 513), (16, 3, 257), (19, 4, 100), (32, 7, 64)])
def test_oracles_match_the_host_and_torch_rules(n, f, d):
  """On tie-free random operands the oracles agree with the host library and the torch rules (fp32 back-ends): the same selections,
  and outputs within the bound of an fp32 sum of the same terms."""
  X = random_operands(n, d, seed=n * 100 + d, byzantine=("scaled",) * f)
  X64, G = X.astype(np.float64), torch.from_numpy(X)
  m = n - f - 2
  everything = np.ones(X.shape, dtype=bool)
  for got in (_ops.host_average(G), _ops.torch_average(G)):
    assert_within(got.numpy(), serial_sum(X64) / n, sum_bound(X64, everything, n), "average")
  for got in (_ops.host_average_nan(G), _ops.torch_average_nan(G)):
    assert_within(got.numpy(), serial_sum(X64) / n, sum_bound(X64, everything, n), "average-nan")
  for got in (_ops.host_median(G), _ops.torch_median(G)):
    assert_bits(got.numpy(), median_ref(X64), "median")
  _, total, keep = averaged_median_ref(X64, n - f, exact=True)
  for got in (_ops.host_averaged_median(G, n - f), _ops.torch_averaged_median(G, n - f)):
    assert_within(got.numpy(), total / (n - f), sum_bound(X64, keep, n - f), "averaged-median")
  _, mask, _, D = krum_ref(X64, f, m)
  _, selected = _ops.host_krum(G, f, m, return_selected=True)
  assert sum(1 << int(i) for i in selected) == mask
  _, selected = _ops.torch_krum(G, f, m, return_selected=True)
  assert sum(1 << int(i) for i in selected) == mask
  assert_distances(_ops.host_pairwise_distances(G).numpy(), D, gamma(d + 2))
  if n >= 4 * f + 3:
    _, masks, _, _, _, _, _ = bulyan_ref(X64, f, m)
    weights = _ops.host_bulyan_weights(_ops.host_pairwise_distances(G), f, m)
    assert masks == [sum(1 << i for i in range(n) if weights[k, i] != 0) for k in range(len(masks))]


@pytest.mark.parametrize("f", range(8))
def test_bulyan_oracle_masks_match_torch_bulyan_weights_on_grid_data(f):
  """The Bulyan oracle, written from DESIGN.md, selects what `_ops.torch_bulyan_weights` selects on grid operands with ties."""
  for n in range(4 * f + 3, 33, 3):
    X = distance_operands(n, f, 40, seed=n + 100 * f).astype(np.float64)
    for m in sorted({n - 2 * f - 2, n - f - 2, n}):
      _, masks, _, D, _, _, _ = bulyan_ref(X, f, m)
      weights = _ops.torch_bulyan_weights(torch.from_numpy(D), f, m)
      assert masks == [sum(1 << i for i in range(n) if weights[k, i] != 0) for k in range(len(masks))], (n, f, m)


def test_oracles_on_hand_computed_cases():
  nan, inf, nz = np.nan, np.inf, -0.0
  # ties -> lower index, -Inf after every finite value, -0 == +0
  X = np.array([[2.0, nz, -inf, 0.0, nan, 1.0],
                [1.0, 0.0, 5.0, nz, nan, 1.0],
                [2.0, nz, -1.0, 0.0, inf, -inf],
                [1.0, 0.0, 7.0, nz, -inf, 3.0]])
  assert_bits(median_ref(X), np.array([2.0, nz, 7.0, 0.0, inf, 3.0], dtype=np.float32))
  assert ranks(X)[:, 0].tolist() == [2, 0, 3, 1] and ranks(X)[:, 1].tolist() == [0, 1, 2, 3]
  # the average of a -0 column is +0; average-nan of a column with no finite value is NaN
  assert_bits(average_ref(np.array([[nz], [nz], [nz]])), np.array([0.0], dtype=np.float32))
  assert_bits(average_nan_ref(X[:, 4:6]), np.array([nan, (1.0 + 1.0 + 3.0) / 3], dtype=np.float32))
  # averaged-median: median 1 of [3, -1, 1, 0, 2]; deviations 2, 2, 0, 1, 1 -> beta = 3 keeps rows 2, 3, 4 (1 + 0 + 2) / 3 = 1
  col = np.array([[3.0], [-1.0], [1.0], [0.0], [2.0]])
  assert_bits(averaged_median_ref(col, 3)[0], np.array([1.0], dtype=np.float32))
  assert_bits(averaged_median_ref(col, 4)[0], np.array([(3.0 + 1.0 + 0.0 + 2.0) / 4], dtype=np.float32))   # the tie 3 / -1 -> row 0
  # a non-finite median makes every deviation non-finite: the first beta rows by index
  assert_bits(averaged_median_ref(np.array([[nan], [1.0], [inf]]), 2)[0], np.array([nan], dtype=np.float32))
  assert_bits(averaged_median_ref(np.array([[1.0], [inf], [inf]]), 1)[0], np.array([1.0], dtype=np.float32))
  # Krum: rows 0 and 1 duplicated, row 3 +Inf. n = 4, f = 0: scores sum the 2 nearest: [0 + 4, 0 + 4, 4 + 4, inf]; m = 2 -> rows 0, 1
  R = np.array([[0.0, 0.0], [0.0, 0.0], [2.0, 0.0], [inf, 1.0]])
  out, mask, scores, D = krum_ref(R, 0, 2)
  assert scores == [4.0, 4.0, 8.0, inf] and mask == 0b0011 and np.isinf(D[3, :3]).all()
  out, mask, _, _ = krum_ref(R, 0, 4)
  assert mask == 0b1111 and np.isinf(out[0])
  # Bulyan, n = 3, f = 0: theta = 1, one round of the m best, beta = 1
  out, masks, means, _, _, _, _ = bulyan_ref(np.array([[0.0], [1.0], [5.0]]), 0, 2)
  assert masks == [0b011] and means.tolist() == [[0.5]] and out.tolist() == [0.5]


# ---------------------------------------------------------------------------- #
# GPU: grid operands, bit for bit

def _coordinate_ds(n):
  tv = threads_vec(n)
  return (1, 3, 4, 5, tv - 4, tv, tv + 4, tv + 1)


@gpu
@pytest.mark.parametrize("n", COORD_N)
@pytest.mark.parametrize("rule", COORD_RULES)
def test_coordinate_rules_bit_exact_on_grid_operands(rule, n, launches):
  """Ties, signed zeros, single and whole-row NaN / +-Inf, columns with more than n / 2 or no finite value; d from 1 to just above
  a multiple of threads x VEC (d % 4 != 0 pads the rows), and once a G view 4 bytes into its allocation."""
  calls = 0
  for s, d in enumerate(_coordinate_ds(n)):
    for bad_rows in (False, True):
      X = coordinate_operands(n, d, seed=1000 * n + 10 * s + bad_rows, bad_rows=bad_rows)
      for beta in (sorted({1, (n + 1) // 2, n}) if rule == "averaged-median" else (0,)):
        out, _, _ = aggregate(spec_of(rule, n, beta=beta), X, offset=(s == 1 and bad_rows))
        calls += 1
        assert_bits(out, reference(rule, X.astype(np.float64), beta=beta)[0], (rule, n, d, bad_rows, beta))
  assert launches == [rule] * calls


def _krum_cases():
  for n in COORD_N:
    for f in sorted({0, n - 3}):
      if n - f - 2 >= 1:
        for m in sorted({1, n - f - 2, n}):
          yield n, f, m


@gpu
@pytest.mark.parametrize("n,f,m", list(_krum_cases()))
def test_krum_bit_exact_on_grid_operands(n, f, m, launches):
  """Duplicated rows (equal distances, equal scores), integer columns; a +Inf row and a NaN-spotted row (distances +inf; never
  selected while enough finite rows remain). Output, every off-diagonal distance, theta = 1 and the mask bit for bit."""
  for s, (d, bad) in enumerate(((7, False), (threads_vec(n) + 4, False), (64, True), (5, True))):
    if bad and n < 4:
      continue
    X = distance_operands(n, f, d, seed=31 * n + 7 * f + m + s, bad=bad)
    out, dist, info = aggregate(spec_of("krum", n, f, m), X, offset=(s == 3))
    want, mask, scores, D = krum_ref(X.astype(np.float64), f, m)
    assert_distances(dist, D)
    assert int(info[0]) == 1 and masks_of(info, 1) == [mask], (bin(masks_of(info, 1)[0]), bin(mask))
    assert_bits(out, want, (n, f, m, d))
    if bad and m <= n - 2 and sum(math.isfinite(v) for v in scores) >= m:
      assert not mask & (1 << 1) and not mask & (1 << (n - 2))
  assert launches and set(launches) == {"krum"}


def _bulyan_cases():
  for f in range(8):
    for n in range(4 * f + 3, 33):
      yield n, f


@gpu
@pytest.mark.parametrize("n,f", list(_bulyan_cases()))
def test_bulyan_on_grid_operands(n, f, launches):
  """Duplicated rows, integer columns, and a +Inf row with a NaN-spotted row (never selected when f >= 1). Masks, theta, every
  off-diagonal distance bit for bit; with n = 4f + 3 (beta = 1) the output is one theta mean, bit for bit;
  otherwise the kernel's fp32 sum of beta theta means, divided once, is within gamma_beta sum |mean| / beta of the exact quotient (the
  means themselves are the oracle's fp32 values: they decide the selection, which is exact)."""
  theta, beta = n - 2 * f - 2, n - 4 * f - 2
  for s, (d, bad, m) in enumerate(((12, False, n - f - 2), (threads_vec(n) - 4, False, theta), (40, True, theta), (9, False, n))):
    X = distance_operands(n, f, d, seed=97 * n + f + s, bad=bad)
    out, dist, info = aggregate(spec_of("bulyan", n, f, m), X)
    want, masks, means, D, _, total, keep = bulyan_ref(X.astype(np.float64), f, m)
    assert_distances(dist, D)
    assert int(info[0]) == theta and masks_of(info, theta) == masks, (masks_of(info, theta), masks)
    if bad and f >= 1:   # n - f - 2 <= n - 3 finite distances score every finite row; the theta - r selected rows are all finite
      assert not any(mask & (1 << 1 | 1 << (n - 2)) for mask in masks)
    if beta == 1:
      assert_bits(out, want, (n, f, m, d))
    else:
      assert_within(out, total / beta, sum_bound(means.astype(np.float64), keep, beta), (n, f, m, d))
  assert launches and set(launches) == {"bulyan"}


@gpu
@pytest.mark.parametrize("n,f,seed", [(7, 1, 3), (11, 2, 5), (19, 4, 2), (32, 7, 1)])
def test_bulyan_subtracts_the_pruned_distance_only(n, f, seed, launches):
  """Operands where a round's best row is one of the f + 1 farthest (pruned) neighbours of a row still present: that row subtracts 0,
  not its distance to the best, and the later rounds select accordingly."""
  X = None
  for attempt in range(200):
    Y = distance_operands(n, f, 8, seed=seed * 1000 + attempt)
    if bulyan_ref(Y.astype(np.float64), f, n - 2 * f - 2)[4]:
      X = Y
      break
  assert X is not None
  out, dist, info = aggregate(spec_of("bulyan", n, f, n - 2 * f - 2), X)
  _, masks, _, D, pruned_best, _, _ = bulyan_ref(X.astype(np.float64), f, n - 2 * f - 2)
  assert pruned_best
  assert_distances(dist, D)
  assert masks_of(info, n - 2 * f - 2) == masks
  assert launches == ["bulyan"]


def _shape_rules():
  for rule in COORD_RULES + ("krum", "bulyan"):
    for n in (1, 2, 3, 8, 9, 16, 17, 32):
      if rule == "krum" and n < 3 or rule == "bulyan" and n < 7:
        continue
      yield rule, n


def _segments(d, count, seed):
  """`count` owned segments of uneven length (multiples of 4) inside [0, d), a gap after each, one of them empty, shuffled."""
  rng = np.random.default_rng(seed)
  p = [0] + (np.sort(rng.choice(np.arange(1, d // 4), size=2 * count - 1, replace=False)) * 4).tolist() + [d]
  segs = [(p[2 * k], p[2 * k + 1]) for k in range(count)]
  segs[count // 2] = (segs[count // 2][0], segs[count // 2][0])   # an empty one
  return [segs[k] for k in rng.permutation(count)]


@gpu
@pytest.mark.parametrize("rule,n", list(_shape_rules()))
def test_launch_shapes_bit_exact(rule, n, launches):
  """Through `FusedLauncher.launch` and `phase_a`: one CTA (the grid-stride loops take many turns) and the full grid, with and without
  a staging tile, 2 to 8 owned segments of uneven length (one empty, not in ascending order, gaps between them), and for Krum and
  Bulyan 1 to nseg - 1 segments pre-accumulated by `phase_a`. agg_out keeps its NaN sentinel outside the owned segments. Everything
  is bit for bit but Bulyan's output with beta > 1, which is held to its bound."""
  f = 0 if rule in COORD_RULES else (n - 3) // 4 if rule == "bulyan" else max(0, n - 4)
  m = n - f - 2 if rule in ("krum", "bulyan") else 0
  beta = (n + 1) // 2 if rule == "averaged-median" else 0
  d = 3 * threads_vec(n) + 12
  if rule in ("krum", "bulyan"):
    X = distance_operands(n, f, d, seed=n + len(rule))
  else:
    X = coordinate_operands(n, d, seed=n + len(rule), bad_rows=True)
  spec = spec_of(rule, n, f, m, beta)
  runs = [dict(max_ctas=1), dict(max_ctas=1, staging=True), dict(), dict(staging=True)]
  for count in (2, 3, 5, 8):
    segs = _segments(d, count, seed=count * 31 + n)
    runs.append(dict(segments=segs, staging=count % 2 == 1, max_ctas=1 if count == 8 else 0))
    if rule in ("krum", "bulyan"):
      for first in sorted({1, count // 2, count - 1}):
        runs.append(dict(segments=segs, staging=first % 2 == 0, first_seg=first, max_ctas=1 if first == 1 else 0))
  for kwargs in runs:
    segs = kwargs.get("segments", [(0, d)])
    cols = owned_columns(d, segs)
    want, masks, D = reference(rule, X[:, cols].astype(np.float64), f, m, beta)
    out, dist, info = launch(spec, X, **kwargs)
    assert_sentinel(out, segs)
    if rule == "bulyan" and spec.beta > 1:   # the beta-average of non-integer theta means: the bound of `test_bulyan_on_grid_operands`
      _, _, means, _, _, total, keep = bulyan_ref(X[:, cols].astype(np.float64), f, m)
      assert_within(out[cols], total / spec.beta, sum_bound(means.astype(np.float64), keep, spec.beta), (rule, n, kwargs))
    else:
      assert_bits(out[cols], want, (rule, n, kwargs))
    if masks is not None:
      assert_distances(dist, D)
      assert int(info[0]) == len(masks) and masks_of(info, len(masks)) == masks, (kwargs, masks_of(info, len(masks)), masks)
  assert launches == [rule] * len(runs)


# ---------------------------------------------------------------------------- #
# GPU: random operands with Byzantine rows, within derived bounds

BYZANTINE = ("scaled", "shifted", "spotted")


@gpu
@pytest.mark.parametrize("n", (3, 8, 9, 17, 32))
@pytest.mark.parametrize("rule", COORD_RULES)
def test_coordinate_rules_on_random_byzantine_operands(rule, n, launches):
  """Median is a selection: bit for bit. The averaged median's fp32 deviations and their ranking are the oracle's exactly, so only
  its sum of the beta kept values, in fp32, and the one division differ: gamma_beta sum |kept| / beta. The average and average-nan
  add their k terms in fp32 and divide once: gamma_k sum |terms| / k."""
  d = 2 * threads_vec(n) + 12
  X = random_operands(n, d, seed=n + 7 * len(rule), byzantine=BYZANTINE[:min(3, n - 1)])
  X64 = X.astype(np.float64)
  beta = max(1, n - 2)
  out, _, _ = aggregate(spec_of(rule, n, beta=beta), X)
  if rule == "median":
    assert_bits(out, median_ref(X64))
  elif rule == "averaged-median":
    _, total, keep = averaged_median_ref(X64, beta, exact=True)
    assert_within(out, total / beta, sum_bound(X64, keep, beta))
  else:
    keep = np.isfinite(X64) if rule == "average-nan" else np.ones(X.shape, dtype=bool)
    count = keep.sum(axis=0)
    with np.errstate(invalid="ignore", divide="ignore"):
      assert_within(out, serial_sum(X64, keep) / count, sum_bound(X64, keep, count))
  assert launches == [rule]


def _assert_margin(values, boundary, rel):
  """The sorted finite values at positions boundary - 1 and boundary are further apart than their bounds: the selection of the first
  `boundary` cannot change under the kernel's rounding."""
  ordered = sorted(values, key=lambda v: order_key([v])[0])
  if 0 < boundary < len(ordered):
    a, b = ordered[boundary - 1], ordered[boundary]
    if math.isfinite(a) and math.isfinite(b):
      assert (1 + rel) * a < (1 - rel) * b, (boundary, a, b)


@gpu
@pytest.mark.parametrize("n,f", [(4, 0), (8, 1), (9, 2), (17, 4), (24, 5), (32, 7)])
def test_krum_on_random_byzantine_operands(n, f, launches):
  """Distances within gamma_(d+2) of the float64 ones, pair by pair; the mask exactly once the case has asserted that the m-th and
  (m+1)-th scores are further apart than their bounds; the mean of the m selected rows within gamma_m sum |x| / m."""
  d = 300
  k = n - f - 2
  for byz in (BYZANTINE[:max(1, f)], ("scaled", "spotted") if f >= 1 else ("scaled",)):
    X = random_operands(n, d, seed=n * 10 + f + len(byz), byzantine=byz)
    X64 = X.astype(np.float64)
    D = distances_ref(X64)
    # a score adds k computed distances, each within gamma_(d+2) of its exact value (d squared differences of one rounded difference
    # each, summed in some tree), in k - 1 fp32 additions: within gamma_(d+2+k) of the exact score. The k smallest computed distances
    # are within the same factor of the k smallest exact ones, whichever rows they are.
    rel = gamma(d + 2 + k)
    for m in sorted({1, k}):
      want, mask, scores, _ = krum_ref(X64, f, m, D)
      _assert_margin(scores, m, rel)
      out, dist, info = aggregate(spec_of("krum", n, f, m), X)
      assert_distances(dist, D, gamma(d + 2))
      assert masks_of(info, 1) == [mask]
      keep = np.zeros(X.shape, dtype=bool)
      keep[[i for i in range(n) if (mask >> i) & 1]] = True
      assert_within(out, serial_sum(X64, keep) / m, sum_bound(X64, keep, m))
  assert launches and set(launches) == {"krum"}


def _surely_scored(D, i, j, k, delta):
  """Whether j is, or is not, among row i's k scored neighbours for every computed matrix within a factor delta of D. A non-finite
  distance is computed exactly (+inf) and ties among them go by index."""
  v = D[i, j]
  if not math.isfinite(v):
    return True
  others = [D[i, o] for o in range(D.shape[0]) if o not in (i, j) and math.isfinite(D[i, o])]
  before = sum(o * (1 + delta) < v * (1 - delta) for o in others)
  unsure = sum(not o * (1 + delta) < v * (1 - delta) and not o * (1 - delta) > v * (1 + delta) for o in others)
  return before + unsure < k or before >= k


def _assert_bulyan_rounds_determined(D, f, m, d):
  """Bulyan's masks are the oracle's for every computed matrix within gamma_(d+2) of D: follows the rounds with an error bound per
  score (gamma_(d+2+k) of the initial sum; each subtraction adds gamma_(d+2) of the distance and one rounding of the result; a
  subtraction that some computed matrix would skip, because the best row is near row i's k-th neighbour, adds the whole distance)
  and asserts that the best row and the first m - r rows of every round are separated from the others by more than the bounds."""
  n = D.shape[0]
  k, theta, delta = n - f - 2, n - 2 * f - 2, gamma(d + 2)
  near = neighbours(D, k)
  scored = [set(near[i][:k]) for i in range(n)]
  score = [sum(float(D[i, j]) for j in near[i][:k]) for i in range(n)]
  err = [gamma(d + 2 + k) * s if math.isfinite(s) else 0.0 for s in score]
  removed = set()
  for r in range(theta):
    present = sorted((i for i in range(n) if i not in removed), key=lambda i: _item_key(score[i], i))
    for cut in (1, m - r):
      last = present[cut - 1]
      if cut < len(present) and math.isfinite(score[last]):
        rest = min(score[j] - err[j] if math.isfinite(score[j]) else math.inf for j in present[cut:])
        assert score[last] + err[last] < rest, (r, cut, score[last], err[last], rest)
    best = present[0]
    removed.add(best)
    for i in present[1:]:
      if not _surely_scored(D, i, best, k, delta):
        err[i] += D[i, best]
      if best in scored[i]:
        score[i] = score[i] - float(D[i, best]) if math.isfinite(score[i]) else math.nan   # +inf - +inf: non-finite either way
        if math.isfinite(score[i]):
          err[i] += delta * D[i, best] + U * abs(score[i])


@gpu
@pytest.mark.parametrize("n,f", [(7, 1), (11, 2), (15, 3), (23, 5), (32, 7)])
def test_bulyan_on_random_byzantine_operands(n, f, launches):
  """Masks exactly once `_assert_bulyan_rounds_determined` holds. Each theta mean of c rows is then within E = gamma_c sum |x| / c;
  the case asserts, per coordinate, that the median of the means is separated from its neighbours by more than 2E and the beta-th
  and (beta+1)-th deviations by more than 4E + 2u |dev|, so the kernel keeps the oracle's means, and its output is within
  gamma_beta sum |kept| / beta + max E of the exact one."""
  d = 300
  theta, beta, m = n - 2 * f - 2, n - 4 * f - 2, n - f - 2
  X = random_operands(n, d, seed=n * 3 + f + 1, byzantine=("scaled", "shifted", "spotted")[:f] if f < 3 else ("scaled",) * (f - 1) + ("spotted",))
  X64 = X.astype(np.float64)
  D = distances_ref(X64)
  _, masks, _, _, _, _, _ = bulyan_ref(X64, f, m, D)
  _assert_bulyan_rounds_determined(D, f, m, d)
  exact_means, errors = [], []
  for mask in masks:
    keep = np.zeros(X.shape, dtype=bool)
    keep[[i for i in range(n) if (mask >> i) & 1]] = True
    count = bin(mask).count("1")
    exact_means.append(serial_sum(X64, keep) / count)
    errors.append(sum_bound(X64, keep, count))
  M, E = np.stack(exact_means), np.max(np.stack(errors), axis=0)
  mid = theta // 2
  if theta > 1:
    assert (np.diff(np.sort(M, axis=0), axis=0)[max(0, mid - 1):mid + 1] > 2 * E).all()
  dev = np.sort(np.abs(M - np.take_along_axis(M, np.argsort(M, axis=0, kind="stable")[mid][None], axis=0)), axis=0)
  if beta < theta:
    assert (dev[beta] - dev[beta - 1] > 4 * E + 2 * U * dev[beta]).all()
  _, total, keep = averaged_median_ref(M, beta, exact=True)
  out, dist, info = aggregate(spec_of("bulyan", n, f, m), X)
  assert_distances(dist, D, gamma(d + 2))
  assert int(info[0]) == theta and masks_of(info, theta) == masks
  assert_within(out, total / beta, sum_bound(M, keep, beta) + E)
  assert launches == ["bulyan"]


# ---------------------------------------------------------------------------- #
# GPU: the reference's stored inputs

@gpu
@pytest.mark.parametrize("n,d", [(4, 50), (7, 1001), (8, 4096), (11, 333)])
def test_kernel_on_the_reference_inputs(n, d, launches):
  """The kernel on the original AggregaThor's stored inputs: its median is the reference's, bit for bit; its average-nan and
  averaged-median are within gamma_k sum |x| / k of the exact quotient, as the reference's own outputs are (a CPU test above)."""
  g = _golden()
  key = "%d_%d_" % (n, d)
  X, clean = g[key + "G"], g[key + "clean"]
  out, _, _ = aggregate(spec_of("median", n), X)
  assert_bits(out, g[key + "median"])
  X64 = X.astype(np.float64)
  finite = np.isfinite(X64)
  out, _, _ = aggregate(spec_of("average-nan", n), X)
  assert_within(out, serial_sum(X64, finite) / finite.sum(axis=0), sum_bound(X64, finite, finite.sum(axis=0)))
  _, total, keep = averaged_median_ref(clean.astype(np.float64), n - 2)
  out, _, _ = aggregate(spec_of("averaged-median", n, beta=n - 2), clean)
  assert_within(out, total / (n - 2), sum_bound(clean.astype(np.float64), keep, n - 2))
  assert launches == ["median", "average-nan", "averaged-median"]

"""Geometric median (smoothed Weiszfeld, RFA) on the host library and the torch reference: a float64 NumPy oracle of the same
definition, exact dyadic cases, excluded non-finite rows, the descent/robustness bound, argument checks and training under attack."""

import math

import numpy as np
import pytest
import torch

from aggregathor_b200 import aggregators, attacks, experiments, tools
from aggregathor_b200.aggregators import FusedSpec, _ops
from aggregathor_b200.engine.trainer import Manager


def _oracle(X, iterations, nu):
  """float64 NumPy Weiszfeld from the upper coordinate-wise median (finite inputs): (z_T, [T, n] distances)."""
  X = np.asarray(X, dtype=np.float64)
  n = X.shape[0]
  z = np.sort(X, axis=0, kind="stable")[n // 2]
  dists = []
  for _ in range(iterations):
    D = ((X - z) ** 2).sum(axis=1)
    dists.append(D)
    kept = np.isfinite(D)
    if not kept.any():
      continue
    beta = 1.0 / np.maximum(nu, np.sqrt(D[kept]))
    z = (beta[:, None] * X[kept]).sum(axis=0) / beta.sum()
  return z, np.array(dists)


def _data(n, d, seed, outliers=0):
  gen = torch.Generator().manual_seed(seed)
  G = torch.randn(n, d, generator=gen)
  for k in range(outliers):
    G[n - 1 - k] = G[n - 1 - k] * 30 + 5
  return G


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("n", list(range(3, 41)))
def test_host_against_float64_oracle(n, dtype):
  d, nu = 257, 1e-6
  f = (n - 1) // 4
  G = _data(n, d, seed=n, outliers=f).to(dtype)
  u = 2.0 ** -24 if dtype == torch.float32 else 2.0 ** -53
  for iterations in (1, 3, 8):
    out, dist = _ops.host_geometric_median(G, iterations, nu, return_distances=True)
    ref, ref_dist = _oracle(G.numpy(), iterations, float(np.float32(nu)))
    assert out.dtype == dtype and dist.shape == (iterations, n)
    # forward error: per iteration, D carries (d + 2) u relative error (beta half of it), the weighted means (n + 2) u; both act on
    # distances of the size of the rows' spread; factor 4 per iteration for the propagation through the next distances
    spread = float(np.abs(G.numpy().astype(np.float64)).max()) * 2
    tol = 4 * (iterations + 1) * ((d + 2) + (n + 2)) * u * spread
    err = float(np.abs(out.numpy().astype(np.float64) - ref).max())
    assert err <= tol, (n, iterations, err, tol)
    assert np.allclose(dist.numpy(), ref_dist, rtol=4 * (iterations + 1) * (d + 2) * u, atol=0)
    torch_out = _ops.torch_geometric_median(G, iterations, nu)
    assert float(np.abs(torch_out.numpy().astype(np.float64) - ref).max()) <= tol


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("pairs,centres", [(1, 1), (3, 1), (3, 2), (7, 1), (15, 2)])
def test_exact_dyadic_cases(pairs, centres, dtype):
  """Rows c (one or two copies) and c +- 2^k e_j: every sqrt(D) is a power of two, so are the weights (nu = 2^-6 below every
  2^k), every product and partial sum is exact, and the symmetric pairs cancel: every iterate is c, bit for bit."""
  d = 40
  gen = torch.Generator().manual_seed(pairs * 10 + centres)
  c = (torch.randint(-32, 33, (d,), generator=gen).to(dtype)) / 4
  rows = [c.clone() for _ in range(centres)]
  for p in range(pairs):
    e = torch.zeros(d, dtype=dtype)
    e[(3 * p) % d] = 2.0 ** (1 + p % 3)
    rows += [c + e, c - e]
  G = torch.stack(rows)
  for iterations in (1, 2, 16):
    out, dist = _ops.host_geometric_median(G, iterations, 2.0 ** -6, return_distances=True)
    assert torch.equal(out, c), (pairs, centres, iterations)
    assert torch.equal(dist[0, :centres], torch.zeros(centres, dtype=dtype))
    assert torch.equal(_ops.torch_geometric_median(G, iterations, 2.0 ** -6), c)


def test_non_finite_rows_are_skipped():
  n, d = 9, 301
  G = _data(n, d, seed=3)
  G[7, 10] = float("nan")
  G[8, ::7] = float("inf")
  G[8, 1::7] = float("-inf")
  for dtype in (torch.float32, torch.float64):
    out, dist = _ops.host_geometric_median(G.to(dtype), 3, 1e-6, return_distances=True)
    assert bool(torch.isfinite(out).all())
    assert not bool(torch.isfinite(dist[:, 7:]).any()) and bool(torch.isfinite(dist[:, :7]).all())
    # the kept rows only, from the same (finite) median of all nine rows
    z0 = _ops.host_median(G.to(dtype)).numpy().astype(np.float64)
    X = G[:7].numpy().astype(np.float64)
    z = z0
    for _ in range(3):
      D = ((X - z) ** 2).sum(axis=1)
      beta = 1.0 / np.maximum(float(np.float32(1e-6)), np.sqrt(D))
      z = (beta[:, None] * X).sum(axis=0) / beta.sum()
    assert float(np.abs(out.numpy() - z).max()) <= 1e-4
    assert torch.allclose(_ops.torch_geometric_median(G.to(dtype), 3, 1e-6), out, rtol=0, atol=1e-4)


def test_no_kept_row_keeps_the_median():
  """A coordinate where every value is NaN makes the median, hence every distance, NaN: no row is ever kept, z_T = z_0."""
  G = _data(6, 50, seed=4)
  G[:, 5] = float("nan")
  for dtype in (torch.float32, torch.float64):
    out, dist = _ops.host_geometric_median(G.to(dtype), 4, 1e-6, return_distances=True)
    median = _ops.host_median(G.to(dtype))
    assert torch.equal(torch.isnan(out), torch.isnan(median))
    assert torch.equal(out[~torch.isnan(out)], median[~torch.isnan(median)])
    assert not bool(torch.isfinite(dist).any())


@pytest.mark.parametrize("scale", [1e1, 1e4, 1e8, 1e16])
@pytest.mark.parametrize("n,b", [(5, 2), (8, 3), (19, 9), (32, 15)])
def test_descent_bound_under_attack(n, b, scale):
  """Smoothed Weiszfeld never increases F(z) = sum_i f_nu(||z - x_i||), with r <= f_nu(r) <= r + nu/2; with b < n/2 rows anywhere
  and c the mean of the h honest rows: (h - b) ||z_T - c|| <= 2 sum_honest ||x_i - c|| + n ||z_0 - c|| + n nu / 2."""
  d, nu = 64, 1e-3
  h = n - b
  gen = torch.Generator().manual_seed(n * 100 + b)
  G = torch.randn(n, d, generator=gen)
  G[h:] = torch.randn(b, d, generator=gen).sign() * scale * (1 + torch.rand(b, d, generator=gen))
  X = G.numpy().astype(np.float64)
  c = X[:h].mean(axis=0)
  rhs_base = 2 * np.linalg.norm(X[:h] - c, axis=1).sum() + n * nu / 2
  for dtype in (torch.float32, torch.float64):
    z0 = _ops.host_median(G.to(dtype)).numpy().astype(np.float64)
    rhs = rhs_base + n * np.linalg.norm(z0 - c)
    for iterations in (1, 3, 16):
      for out in (_ops.host_geometric_median(G.to(dtype), iterations, nu), _ops.torch_geometric_median(G.to(dtype), iterations, nu)):
        lhs = (h - b) * np.linalg.norm(out.numpy().astype(np.float64) - c)
        assert lhs <= rhs * (1 + 1e-4) + 1e-4, (n, b, scale, iterations, lhs, rhs)


def test_argument_errors():
  with pytest.raises(tools.UserException):
    aggregators.instantiate("geometric-median", 8, 4, [])
  with pytest.raises(tools.UserException):
    aggregators.instantiate("geometric-median", 8, -1, [])
  for args in (["iterations:0"], ["iterations:17"], ["iterations:2.5"], ["nu:0"], ["nu:-1"], ["nu:inf"], ["nu:nan"], ["nu:1e-50"], ["nu:1e39"], ["nu:x"]):
    with pytest.raises(tools.UserException):
      aggregators.instantiate("geometric-median", 8, 2, args)
  gar = aggregators.instantiate("geometric-median", 8, 3, ["iterations:16", "nu:0.1"])
  spec = gar.fused_spec()
  assert (spec.rule, spec.n, spec.f, spec.iterations) == ("geometric-median", 8, 3, 16)
  assert spec.nu == float(np.float32(0.1)) and spec.rule_id == 8
  assert FusedSpec("krum", 8, 2, 4).rule_id == 4 and "iterations" not in repr(FusedSpec("krum", 8, 2, 4))
  G = _data(8, 10, seed=1)
  with pytest.raises(tools.UserException):
    _ops.host_geometric_median(G, 0, 1e-6)
  with pytest.raises(tools.UserException):
    _ops.torch_geometric_median(G, 3, 0.0)


def test_plugin_dispatch_on_cpu():
  G = _data(7, 500, seed=8, outliers=2)
  gar = aggregators.instantiate("geometric-median", 7, 2, ["iterations:4"])
  out = gar.aggregate(list(G))
  assert torch.equal(out, _ops.host_geometric_median(G, 4, 1e-6))
  assert torch.equal(gar.aggregate(G.double()), _ops.host_geometric_median(G.double(), 4, 1e-6))


def _manager(gar_name, n, f, attack=None, real=0):
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate(gar_name, n, f, [])
  return Manager(experiment, gar, n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu", attack=attack, nb_real_byz=real)


def test_training_survives_flip_where_average_does_not():
  robust = _manager("geometric-median", 7, 2, attacks.instantiate("flip", 7, 2, ["factor:-50"]), 2)
  first = float(robust.train())
  for _ in range(25):
    last = float(robust.train())
  assert last == last and last < first
  assert robust.evaluate()["top1-X-acc"] > 0.5
  naive = _manager("average", 7, 2, attacks.instantiate("flip", 7, 2, ["factor:-50"]), 2)
  for _ in range(25):
    loss = float(naive.train())
  assert not (loss == loss and naive.evaluate()["top1-X-acc"] > 0.5 and loss < first)

"""Centered clipping on the host library and the torch reference: an fp32 NumPy replay of the definition from the library's own
distances, a float64 oracle, hand cases, the center carried over calls, argument checks and checkpoint / resume of the center."""

import numpy as np
import pytest
import torch

from aggregathor_b200 import aggregators, experiments, tools
from aggregathor_b200.aggregators import FusedSpec, _ops
from aggregathor_b200.engine.flat import FlatLayout
from aggregathor_b200.engine.optimizers import optimizers
from aggregathor_b200.engine.schedules import build
from aggregathor_b200.engine.trainer import Manager
from aggregathor_b200.parallel.aggregation import HostAggregation


def _data(n, d, seed, outliers=0):
  gen = torch.Generator().manual_seed(seed)
  G = torch.randn(n, d, generator=gen)
  for k in range(outliers):
    G[n - 1 - k] = G[n - 1 - k] * 30 + 5
  return G


def _replay(X, z, dists, tau):
  """The definition in NumPy fp32 (correctly rounded sqrt and division, no FMA) from the given distances [T, n]."""
  one, tau, count = np.float32(1), np.float32(tau), np.float32(X.shape[0])
  for D in dists:
    kept = [i for i in range(X.shape[0]) if np.isfinite(D[i])]
    if not kept:
      continue
    u = np.zeros_like(z)
    for i in kept:
      s = np.sqrt(np.float32(D[i]))
      c = one if s <= tau else np.float32(tau / s)
      u = u + c * (X[i] - z)
    z = z + u / count
  return z


def _oracle(X, z, iterations, tau):
  """float64 NumPy centered clipping (finite inputs): (z_T, [T, n] distances)."""
  X, z = np.asarray(X, dtype=np.float64), np.asarray(z, dtype=np.float64)
  dists = []
  for _ in range(iterations):
    D = ((X - z) ** 2).sum(axis=1)
    dists.append(D)
    s = np.sqrt(D)
    c = np.where(s <= tau, 1.0, tau / np.maximum(s, 1e-300))
    z = z + (c[:, None] * (X - z)).sum(axis=0) / X.shape[0]
  return z, np.array(dists)


@pytest.mark.parametrize("n", [3, 4, 8, 9, 17, 32, 33])
def test_host_replays_its_own_distances_bit_for_bit(n):
  d, tau = 1003, 3.0
  G = _data(n, d, seed=n, outliers=max(1, n // 4))
  G[0, 17] = float("nan")
  X = G.numpy()
  for iterations in (1, 3, 16):
    center = torch.zeros(d)
    z = np.zeros(d, dtype=np.float32)
    for call in range(3):
      out, dist = _ops.host_centered_clipping(G + call, iterations, tau, center, return_distances=True)
      z = _replay(X + np.float32(call), z, dist.numpy(), tau)
      assert torch.equal(out, torch.from_numpy(z)) and torch.equal(center, out), (n, iterations, call)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("n", list(range(3, 41)))
def test_host_against_float64_oracle(n, dtype):
  d, tau = 257, 4.0
  f = (n - 1) // 4
  G = _data(n, d, seed=n, outliers=f).to(dtype)
  u = 2.0 ** -24 if dtype == torch.float32 else 2.0 ** -53
  for iterations in (1, 3, 8):
    z0 = (torch.randn(d, generator=torch.Generator().manual_seed(n)) * 0.5).to(dtype)
    center = z0.clone()
    out, dist = _ops.host_centered_clipping(G, iterations, tau, center, return_distances=True)
    ref, ref_dist = _oracle(G.numpy(), z0.numpy(), iterations, float(np.float32(tau)))
    # forward error: per iteration D carries (d + 2) u relative error (sqrt and the clipping factor half of it more), the clipped
    # sum (n + 3) u relative to the sum of |x_i - z|, of the size of the rows' spread; factor 4 per iteration for the propagation
    spread = float(np.abs(G.numpy().astype(np.float64)).max()) * 2 + float(np.abs(z0.numpy()).max())
    tol = 4 * (iterations + 1) * ((d + 2) + (n + 3)) * u * spread
    err = float(np.abs(out.numpy().astype(np.float64) - ref).max())
    assert err <= tol, (n, iterations, err, tol)
    assert np.allclose(dist.numpy(), ref_dist, rtol=4 * (iterations + 1) * (d + 2) * u, atol=0)
    torch_center = z0.clone()
    torch_out = _ops.torch_centered_clipping(G, iterations, tau, torch_center)
    assert float(np.abs(torch_out.numpy().astype(np.float64) - ref).max()) <= tol
    assert torch.equal(torch_center, torch_out)


def test_large_tau_single_iteration_is_the_mean_step():
  """tau above every distance, T = 1: every c_i = 1, z_1 = v + (sum (x_i - v)) / n, the sum in ascending order."""
  n, d = 6, 200
  G = _data(n, d, seed=2)
  v = torch.randn(d, generator=torch.Generator().manual_seed(3))
  for dtype in (torch.float32, torch.float64):
    center = v.to(dtype).clone()
    out = _ops.host_centered_clipping(G.to(dtype), 1, 1e30, center)
    total = torch.zeros(d, dtype=dtype)
    for i in range(n):
      total = total + (G[i].to(dtype) - v.to(dtype))
    expect = v.to(dtype) + total / n
    assert torch.equal(out, expect) and torch.equal(center, expect)
    assert torch.equal(_ops.torch_centered_clipping(G.to(dtype), 1, 1e30, v.to(dtype).clone()), expect)


def test_non_finite_rows_are_skipped():
  n, d = 7, 301
  G = _data(n, d, seed=3)
  G[5, 10] = float("nan")
  G[6, ::7] = float("inf")
  G[6, 1::7] = float("-inf")
  for dtype in (torch.float32, torch.float64):
    out, dist = _ops.host_centered_clipping(G.to(dtype), 3, 2.0, torch.zeros(d, dtype=dtype), return_distances=True)
    assert bool(torch.isfinite(out).all())
    assert not bool(torch.isfinite(dist[:, 5:]).any()) and bool(torch.isfinite(dist[:, :5]).all())
    # the five kept rows only, each step divided by all seven rows
    X, z = G[:5].numpy().astype(np.float64), np.zeros(d)
    for _ in range(3):
      s = np.sqrt(((X - z) ** 2).sum(axis=1))
      c = np.where(s <= 2.0, 1.0, 2.0 / s)
      z = z + (c[:, None] * (X - z)).sum(axis=0) / n
    assert float(np.abs(out.numpy() - z).max()) <= 1e-5
    assert torch.allclose(_ops.torch_centered_clipping(G.to(dtype), 3, 2.0, torch.zeros(d, dtype=dtype)), out, rtol=0, atol=1e-5)
  G[:, 4] = float("nan")   # every distance is NaN: no row is kept, the center stays
  center = torch.full((d,), 0.25)
  out = _ops.host_centered_clipping(G, 4, 2.0, center)
  assert torch.equal(out, torch.full((d,), 0.25)) and torch.equal(center, out)


def test_center_carries_over_calls():
  n, d = 5, 64
  G = _data(n, d, seed=9)
  gar = aggregators.instantiate("centered-clipping", n, 1, ["iterations:2", "tau:0.5"])
  center = torch.zeros(d)
  outs = [gar.aggregate(G) for _ in range(3)]
  for k in range(3):
    expect = _ops.host_centered_clipping(G, 2, 0.5, center)
    assert torch.equal(outs[k], expect), k
  assert not torch.equal(outs[0], outs[2])
  mine = torch.zeros(d)
  out = gar.aggregate(G, center=mine)
  assert torch.equal(out, mine) and torch.equal(out, _ops.host_centered_clipping(G, 2, 0.5, torch.zeros(d)))


def test_argument_errors():
  with pytest.raises(tools.UserException):
    aggregators.instantiate("centered-clipping", 8, 4, [])
  with pytest.raises(tools.UserException):
    aggregators.instantiate("centered-clipping", 8, -1, [])
  for args in (["iterations:0"], ["iterations:17"], ["iterations:2.5"], ["tau:0"], ["tau:-1"], ["tau:inf"], ["tau:nan"], ["tau:1e-50"], ["tau:1e39"], ["tau:x"]):
    with pytest.raises(tools.UserException):
      aggregators.instantiate("centered-clipping", 8, 2, args)
  gar = aggregators.instantiate("centered-clipping", 8, 3, [])
  spec = gar.fused_spec()
  assert (spec.rule, spec.n, spec.f, spec.iterations, spec.tau, spec.rule_id) == ("centered-clipping", 8, 3, 1, 10.0, 9)
  spec = aggregators.instantiate("centered-clipping", 8, 3, ["iterations:16", "tau:0.1"]).fused_spec()
  assert spec.iterations == 16 and spec.tau == float(np.float32(0.1))
  assert repr(spec) == "FusedSpec(rule='centered-clipping', n=8, f=3, m=0, beta=0, iterations=16, tau=%r)" % float(np.float32(0.1))
  assert repr(FusedSpec("geometric-median", 8, 2)) == "FusedSpec(rule='geometric-median', n=8, f=2, m=0, beta=0, iterations=3, nu=1e-06)"
  assert "tau" not in repr(FusedSpec("krum", 8, 2, 4))
  G = _data(8, 10, seed=1)
  with pytest.raises(tools.UserException):
    _ops.host_centered_clipping(G, 0, 1.0, torch.zeros(10))
  with pytest.raises(tools.UserException):
    _ops.host_centered_clipping(G, 1, 1.0, torch.zeros(11))
  with pytest.raises(tools.UserException):
    _ops.torch_centered_clipping(G, 3, 0.0, torch.zeros(10))


def test_host_engine_checkpoints_the_center():
  layout = FlatLayout()
  layout.add("w", (50, 3))
  layout.freeze()
  gar = aggregators.instantiate("centered-clipping", 4, 1, ["iterations:2", "tau:0.3"])
  gen = torch.Generator().manual_seed(4)
  grads = [torch.randn(4, layout.padded_size, generator=gen) for _ in range(4)]

  def engine():
    return HostAggregation(gar, layout, 4, build(optimizers, "optimizer", "sgd", []), device="cpu")
  straight = engine()
  for G in grads:
    straight.grads.copy_(G)
    straight.step(0.1)
  first = engine()
  for G in grads[:2]:
    first.grads.copy_(G)
    first.step(0.1)
  state = first.state_dict()
  resumed = engine()
  resumed.params.copy_(first.params)
  resumed.load_state_dict(state)
  assert torch.equal(resumed.center, first.center)
  for G in grads[2:]:
    resumed.grads.copy_(G)
    resumed.step(0.1)
  assert torch.equal(resumed.params, straight.params) and torch.equal(resumed.center, straight.center)


def test_manager_checkpoint_without_a_center_starts_from_zero(monkeypatch):
  warnings = []
  monkeypatch.setattr(tools, "warning", lambda message, *args, **kwargs: warnings.append(message))
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  mgr = Manager(experiment, aggregators.instantiate("centered-clipping", 3, 1, []), 3, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu")
  mgr.train()
  assert bool(mgr.aggregation.center.any())
  state = mgr.state_dict()
  del state["aggregation"]["rule_state"]
  mgr.load_state_dict(state)
  assert not bool(mgr.aggregation.center.any()) and any("center" in w for w in warnings)

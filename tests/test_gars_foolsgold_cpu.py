"""FoolsGold (`aggregators/foolsgold.py`) on the CPU: the shared coefficient arithmetic against a literal float64 transcription of the
paper's Algorithm 1, the host and torch back-ends over consecutive calls on one history, Sybil rows, invariances, argument checks,
checkpoint / resume of the histories, and a label-flipping run whose weights are reported."""

import math

import numpy as np
import pytest
import torch

from aggregathor_b200 import aggregators, attacks, experiments, tools
from aggregathor_b200.aggregators import FusedSpec, _ops
from aggregathor_b200.engine.trainer import Manager


def _equal_bits(a, b):
  a, b = torch.as_tensor(a).cpu().contiguous(), torch.as_tensor(b).cpu().contiguous()
  assert a.dtype == b.dtype and a.shape == b.shape
  view = torch.int64 if a.dtype == torch.float64 else torch.int32
  assert torch.equal(a.view(view), b.view(view))


def _oracle(P, N, bad, kappa):
  """Algorithm 1 of the paper, literal double loops in float64, with this project's policies (zero or non-finite norms, bad rows,
  all-zero weights) -> (alpha, c as float32)."""
  n = len(N)
  P = [[float(P[i][j]) for j in range(n)] for i in range(n)]
  N = [float(x) for x in N]
  usable = [math.isfinite(x) and x != 0.0 for x in N]
  cs = [[0.0] * n for _ in range(n)]
  for i in range(n):
    for j in range(n):
      if i != j and usable[i] and usable[j]:
        q = P[i][j] / (math.sqrt(N[i]) * math.sqrt(N[j]))
        cs[i][j] = q if math.isfinite(q) else 0.0
  v = [max(cs[i]) for i in range(n)]
  for i in range(n):
    for j in range(n):
      if i != j and v[j] > v[i]:
        cs[i][j] = cs[i][j] * v[i] / v[j]
  alpha = [min(max(1.0 - max(cs[i]), 0.0), 1.0) for i in range(n)]
  top = max(alpha)
  if top == 0.0:
    return [0.0] * n, np.zeros(n, dtype=np.float32)
  alpha = [a / top for a in alpha]
  alpha = [0.99 if a == 1.0 else a for a in alpha]
  for i in range(n):
    logit = math.log(alpha[i] / (1.0 - alpha[i])) if alpha[i] > 0.0 else -math.inf
    alpha[i] = min(max(kappa * (logit + 0.5), 0.0), 1.0)
    if bad[i] or not math.isfinite(N[i]):
      alpha[i] = 0.0
  total = 0.0
  for a in alpha:
    total += a
  c = np.array([a / total if total != 0.0 else 0.0 for a in alpha], dtype=np.float64).astype(np.float32)
  return alpha, c


def _sums(H):
  """float32 sums of the rows of H (a history), computed in float64 then rounded: a hand-made input for the coefficient functions."""
  H = np.asarray(H, dtype=np.float64)
  P = (H @ H.T).astype(np.float32)
  return P, np.diagonal(P).copy()


def _hand_made():
  rng = np.random.default_rng(3)
  base = rng.standard_normal((6, 40))
  pardon = base.copy()
  pardon[1] = pardon[0] + 0.05 * rng.standard_normal(40)   # 0 and 1 nearly collinear: v_0, v_1 close to 1
  pardon[2] = pardon[0] + 1.5 * rng.standard_normal(40)    # 2 half-aligned with 0: v_2 < v_0, pardoned
  zero = base.copy()
  zero[3] = 0.0
  # identical histories: cs_ij = N / (sqrt(N) sqrt(N)) is 1 only up to the rounding of the square roots, so these rows have an exact
  # square root (N = 16); otherwise every alpha_i can come out as the same few ulps and be rescaled to 1
  same = np.zeros((5, 40))
  same[:, :16] = np.sign(base[0, :16])
  return {"pardoning": (pardon, np.zeros(6, bool), 1.0), "zero-row": (zero, np.zeros(6, bool), 1.0),
          "identical": (same, np.zeros(5, bool), 1.0), "bad-row": (base, np.array([0, 0, 1, 0, 0, 0], bool), 1.0),
          "kappa-0.25": (pardon, np.zeros(6, bool), 0.25), "kappa-3": (base, np.zeros(6, bool), 3.0), "n=1": (base[:1], np.zeros(1, bool), 1.0)}


@pytest.mark.parametrize("case", list(_hand_made()))
def test_coefficients_match_the_literal_algorithm(case):
  H, bad, kappa = _hand_made()[case]
  P, N = _sums(H)
  alpha, S, c = _ops.foolsgold_coefficients(P, N, bad, kappa)
  want_alpha, want_c = _oracle(P, N, bad, kappa)
  assert np.array_equal(alpha, np.array(want_alpha)) and np.array_equal(c, want_c) and c.dtype == np.float32
  if case == "pardoning":   # the pardon changes row 2's largest similarity
    cs = P.astype(np.float64) / np.sqrt(np.outer(N.astype(np.float64), N.astype(np.float64)))
    np.fill_diagonal(cs, 0.0)
    assert cs.max(axis=1)[0] > cs.max(axis=1)[2] and c[2] > 0
  if case == "zero-row":
    assert c[3] > 0   # a zero history is similar to nobody
  if case == "identical":
    assert not c.any() and S == 0.0
    G = torch.from_numpy(H).float()
    out = _ops.host_foolsgold(G, torch.zeros_like(G))
    assert torch.equal(out, torch.zeros_like(out)) and not torch.signbit(out).any()
  if case == "bad-row":
    assert c[2] == 0 and (c[[0, 1, 3, 4, 5]] > 0).all()
  if case == "n=1":
    assert c.tolist() == [1.0]


def _rows(n, d, seed, nan=False):
  gen = torch.Generator().manual_seed(seed)
  mu = torch.randn(d, generator=gen)
  G = 0.3 * mu + torch.randn((n, d), generator=gen)
  if nan and n > 1:
    G[1, 5] = float("nan")
    G[n - 1, d // 2] = float("-inf")
  return G


def _check_sums(P, H):
  H = H.double().numpy()
  norms = np.linalg.norm(H, axis=1)
  assert np.all(np.abs(P.astype(np.float64) - H @ H.T) <= 1e-5 * np.outer(norms, norms) + 1e-30)


@pytest.mark.parametrize("n", list(range(1, 33)))
def test_host_and_torch_over_consecutive_calls(n):
  d = 517
  Hh, Ht, Hs = torch.zeros(n, d), torch.zeros(n, d), torch.zeros(n, d)
  for call in range(4):
    G = _rows(n, d, 100 * n + call, nan=(call == 2))
    want = Hh + torch.where(torch.isfinite(G), G, torch.zeros_like(G))
    out_h, P, N, bad, c = _ops.host_foolsgold(G, Hh, return_details=True)
    out_t, _, _, _, ct = _ops.torch_foolsgold(G, Ht, sums=(P, N, bad), return_details=True)
    _equal_bits(Hh, want)
    _equal_bits(Ht, want)
    _equal_bits(out_h, out_t)
    assert np.array_equal(c, ct) and c.dtype == np.float32
    assert np.array_equal(bad, ~torch.isfinite(G).all(dim=1).numpy())
    _check_sums(P, Hh)
    own = _ops.torch_foolsgold(G, Hs, return_details=True)   # the torch reference's own sums
    _equal_bits(Hs, want)
    _check_sums(own[1], Hs)
    assert bool(torch.isfinite(out_h).all())
    if c.any():
      assert abs(float(c.astype(np.float64).sum()) - 1.0) <= 1e-6 * n


def test_double_rows():
  G = _rows(5, 300, 1).double()
  H1, H2 = torch.zeros_like(G), torch.zeros_like(G)
  for _ in range(3):
    out_h, P, N, bad, c = _ops.host_foolsgold(G, H1, return_details=True)
    out_t = _ops.torch_foolsgold(G, H2, sums=(P, N, bad))
    assert out_h.dtype == torch.float64 and c.dtype == np.float64 and torch.equal(out_h, out_t) and torch.equal(H1, H2)


def test_sybils_get_no_weight():
  n, k = 10, 3
  byz = list(range(n - k, n))
  gar = aggregators.instantiate("foolsgold", n, k, [])
  alie = attacks.instantiate("alie", n, k, [])
  H = torch.zeros(n, 2000)
  for step in range(5):
    G = _rows(n, 2000, 40 + step)
    _ops.torch_craft_byzantine_(G, byz, "alie", alie.coef)
    assert torch.equal(G[n - 1], G[n - 2]) and torch.equal(G[n - 1], G[n - 3])
    out, P, N, bad, c = _ops.host_foolsgold(G, H, gar.confidence, return_details=True)
    assert (c[byz] == 0).all() and (c[:n - k] > 0).all(), (step, c)


def test_invariances():
  n, d = 7, 640
  G = _rows(n, d, 9)
  out, P, N, bad, c = _ops.host_foolsgold(G, torch.zeros(n, d), return_details=True)
  out4, P4, N4, bad4, c4 = _ops.host_foolsgold(G * 4, torch.zeros(n, d), return_details=True)
  assert np.array_equal(P4, P * 16) and np.array_equal(c4, c)
  _equal_bits(out4, out * 4)
  perm = [3, 0, 6, 1, 5, 2, 4]
  G[2, 11] = float("nan")
  outp, Pp, Np, badp, cp = _ops.host_foolsgold(G[perm], torch.zeros(n, d), return_details=True)
  out, P, N, bad, c = _ops.host_foolsgold(G, torch.zeros(n, d), return_details=True)
  assert np.array_equal(Pp, P[np.ix_(perm, perm)]) and np.array_equal(Np, N[perm]) and np.array_equal(badp, bad[perm])
  assert np.array_equal(_ops.foolsgold_coefficients(Pp, Np, badp, 1.0)[0], _ops.foolsgold_coefficients(P, N, bad, 1.0)[0][perm])
  assert np.allclose(cp, c[perm], rtol=1e-6, atol=0) and cp[perm.index(2)] == 0


def test_rule_ids_and_spec():
  assert FusedSpec.RULES.index("foolsgold") == 13 and FusedSpec.RULES.index("fltrust") == 12
  assert "foolsgold" not in FusedSpec.RULES_WITH_F
  gar = aggregators.instantiate("foolsgold", 8, 2, ["confidence:2.5"])
  spec = gar.fused_spec()
  assert (spec.rule, spec.n, spec.rule_id, spec.confidence, gar.confidence, gar.needs_history) == ("foolsgold", 8, 13, 2.5, 2.5, True)
  assert spec.with_rows(4).confidence == 2.5
  assert aggregators.instantiate("foolsgold", 8, 7, []).confidence == 1.0


def test_argument_errors():
  for args in (["confidence:0"], ["confidence:-1"], ["confidence:nan"], ["confidence:inf"], ["confidence:x"]):
    with pytest.raises(tools.UserException):
      aggregators.instantiate("foolsgold", 8, 2, args)
  with pytest.raises(tools.UserException):
    aggregators.instantiate("foolsgold", 4, 4, [])
  with pytest.raises(tools.UserException, match="history"):
    _ops.torch_foolsgold(torch.ones(4, 8), torch.zeros(4, 9))
  gar = aggregators.instantiate("foolsgold", 4, 1, [])
  G = _rows(4, 32, 2)
  first = gar.aggregate(G)   # a history kept by the object
  assert torch.equal(gar._history, G) and torch.equal(first, _ops.host_foolsgold(G, torch.zeros(4, 32)))


@pytest.mark.parametrize("mix", ["nnm", "arc", "arc+nnm", "bucketing"])
def test_pre_aggregation_is_refused(mix):
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate("foolsgold", 4 if mix == "bucketing" else 8, 2 if mix != "bucketing" else 1, [])
  with pytest.raises(tools.UserException, match="pre-aggregation"):
    Manager(experiment, gar, 8, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu", pre_aggregation=mix,
            bucket_size=2 if mix == "bucketing" else None)


def _manager(n=4, f=1, attack=None, real=0, seed=None):
  experiment = experiments.instantiate("mnist", ["batch-size:16"] + (["seed:%d" % seed] if seed is not None else []))
  gar = aggregators.instantiate("foolsgold", n, f, [])
  return Manager(experiment, gar, n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu", attack=attack, nb_real_byz=real)


def _advance(mgr, steps):
  for stream in mgr.streams:
    for _ in range(steps):
      next(stream)


def test_checkpoint_and_resume_is_bit_identical(monkeypatch):
  straight = _manager()
  assert straight.aggregation.name == "host" and straight.aggregation.history.shape == (4, straight.layout.padded_size)
  for _ in range(6):
    straight.train()
  first = _manager()
  for _ in range(3):
    first.train()
  state = first.state_dict()
  assert state["aggregation"]["rule_state"].shape == (4, first.layout.padded_size)
  resumed = _manager()
  resumed.load_state_dict(state)
  _advance(resumed, 3)   # the input streams restart with the process: skip the batches the first run consumed
  for _ in range(3):
    resumed.train()
  _equal_bits(resumed.params, straight.params)
  _equal_bits(resumed.aggregation.history, straight.aggregation.history)
  # a checkpoint without an [n, d] history restores zero histories, with a warning
  warnings = []
  monkeypatch.setattr(tools, "warning", lambda message, *args, **kwargs: warnings.append(message))
  del state["aggregation"]["rule_state"]
  resumed.load_state_dict(state)
  assert not bool(resumed.aggregation.history.any()) and any("history" in w for w in warnings)


def test_label_flip_weights_are_reported():
  """Whether FoolsGold separates label-flipping workers on mnist has not been established: this run reports the mean weights of the
  flipped and honest workers (`-s` shows them) and checks only that they are weights."""
  n, k = 8, 2
  mgr = _manager(n, k, attacks.instantiate("label-flip", n, k, []), k, seed=1)
  flipped, honest = [], []
  for _ in range(20):
    mgr.train()
    H = mgr.aggregation.history
    P, N = _sums(H.numpy())
    c = _ops.foolsgold_coefficients(P, N, np.zeros(n, bool), mgr.aggregation.gar.confidence)[2]
    assert bool(torch.isfinite(mgr.params).all()) and (c >= 0).all() and (not c.any() or abs(float(c.sum()) - 1) < 1e-5)
    flipped.append(float(c[n - k:].mean()))
    honest.append(float(c[:n - k].mean()))
  print("label-flip on mnist, n = 8, 2 flipped, seed 1, 20 steps: mean c of the flipped workers %.4f, of the honest workers %.4f"
        % (np.mean(flipped), np.mean(honest)))

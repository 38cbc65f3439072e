"""fang-krum and fang-trim (Fang, Cao, Jia & Gong, USENIX Security 2020) on the CPU: the gamma search against an independent brute
force over crafted matrices and hand cases, fang-trim's intervals, draws and a per-coordinate pure-Python transcription, the argument
checks, the host engine end to end and the runner CLI."""

import math
import os
import pathlib
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from aggregathor_b200 import aggregators, attacks, experiments, tools
from aggregathor_b200.aggregators import _ops
from aggregathor_b200.engine.trainer import Manager
from aggregathor_b200.ops import gar as gar_ops

ROOT = pathlib.Path(__file__).resolve().parent.parent
LOCAL = ["--server", '{"local": ["127.0.0.1:7000"]}', "--ps-job-name", "local", "--wk-job-name", "local", "--ev-job-name", "local", "--no-wait"]


def _bits(t):
  return t.detach().cpu().contiguous().view(torch.int32)


def _equal_values(a, b):
  """Equal bit for bit, except that any NaN matches any NaN (same positions)."""
  nan = torch.isnan(a)
  assert torch.equal(nan, torch.isnan(b))
  assert torch.equal(_bits(a)[~nan], _bits(b)[~nan])


# ---------------------------------------------------------------------------- #
# fang-krum: the search

def _krum_winner(X, f):
  """Slot Krum ranks first on the float64 rows X: ascending score (the n - f - 2 smallest distances), ties to the lower slot."""
  n = X.shape[0]
  D = ((X[:, None, :] - X[None, :, :]) ** 2).sum(axis=2)
  scores = [np.sort(np.delete(D[i], i))[:n - f - 2].sum() for i in range(n)]
  return min(range(n), key=lambda i: (scores[i], i))


def _brute_force(G, slots, f, threshold):
  """(gamma, selected) from the crafted float64 matrices of every candidate, gamma_max recomputed from the rows with numpy."""
  n = G.shape[0]
  K, H = len(slots), n - len(slots)
  honest = np.array([G[i].numpy() for i in range(n) if i not in slots], dtype=np.float64)
  mu = _ops._honest_mean([G[i] for i in range(n) if i not in slots], _ops._scalar(G)).numpy().astype(np.float64)
  p = np.sign(mu)
  C = float((p * p).sum())
  dist = np.sqrt(((honest[:, None, :] - honest[None, :, :]) ** 2).sum(axis=2))
  R = [np.sort(np.delete(dist[i], i))[:H - 2].sum() for i in range(H)]
  gamma_max = min(R) / ((n - 2 * K - 1) * math.sqrt(C)) + max(np.sqrt((honest ** 2).sum(axis=1))) / math.sqrt(C)
  last = None
  for t in range(64):
    gamma = gamma_max * 2.0 ** -t
    if t > 0 and gamma < threshold:
      break
    last = gamma
    X = G.numpy().astype(np.float64).copy()
    X[slots] = -gamma * p
    if _krum_winner(X, f) in slots:
      return gamma, True
  return last, False


def _integer_rows(n, d, seed):
  """Small integers around a common offset: every fp32 sum of the statistics is exact, the mean has definite signs."""
  gen = torch.Generator().manual_seed(seed)
  offset = torch.randint(-3, 4, (1, d), generator=gen)
  return (offset + torch.randint(-4, 5, (n, d), generator=gen)).float()


def _search_cases():
  for n in (4, 5, 7, 8, 11, 16, 23, 32):
    for K in sorted({1, (n - 1) // 4, (n - 2) // 2}):
      if K < 1 or n - 2 * K - 1 < 1:
        continue
      for f in sorted({K, max(0, K - 1), (n - 3) // 2}):
        if n - f - 2 >= 1:
          yield n, K, f


@pytest.mark.parametrize("n,K,f", list(_search_cases()))
def test_gamma_matches_a_brute_force_over_crafted_matrices(n, K, f):
  for seed in range(3):
    G = _integer_rows(n, 24, seed=n * 100 + K * 10 + f + seed)
    slots = list(range(n - K, n)) if seed != 1 else list(range(K))   # the Byzantine slots first too
    crafted = G.clone()
    gamma, selected, t, gamma_max, A, B, C, T = _ops.torch_craft_byzantine_(crafted, slots, "fang-krum", f=f, return_details=True)
    assert (gamma, selected, t, gamma_max) == _ops.fang_krum_gamma(A, B, C, T, n, f, slots, _ops.FANG_THRESHOLD)
    expected_gamma, expected_selected = _brute_force(G, slots, f, _ops.fp32(_ops.FANG_THRESHOLD))
    assert selected == expected_selected, (n, K, f, seed)
    assert abs(gamma - expected_gamma) <= 1e-6 * expected_gamma, (gamma, expected_gamma)
    assert gamma == _ops.fp32(gamma_max * 2.0 ** -t)
    p = _ops._sign(_ops._honest_mean([G[i] for i in range(n) if i not in slots], _ops._scalar(G)))
    for i in range(n):
      assert torch.equal(_bits(crafted[i]), _bits(torch.neg(torch.tensor(gamma)) * p if i in slots else G[i]))
    if selected:   # Krum on the crafted fp32 rows picks a Byzantine row
      _, chosen = _ops.torch_krum(crafted, f, 1, return_selected=True)
      assert int(chosen[0]) in slots


def test_gamma_max_hand_case_not_selected():
  """Honest values 1, 2, 3, 4 (d = 1), one Byzantine row, f = 1: mu > 0, C = 1, R = (3, 2, 2, 3), gamma_max = 2 / 2 + 4 = 5. Krum never
  picks -gamma (its two nearest honest values are at least 1 and 2 away, while row 2 scores 1 + 1): the candidates halve down to the
  last one >= 1e-5, 5 * 2^-18."""
  G = torch.tensor([[1.0], [2.0], [3.0], [4.0], [9.0]])
  gamma, selected, t, gamma_max, A, B, C, T = _ops.torch_craft_byzantine_(G, [4], "fang-krum", f=1, return_details=True)
  assert (A, B, C, T) == ([1.0, 4.0, 9.0, 16.0], [1.0, 2.0, 3.0, 4.0], 1.0, [1.0, 4.0, 9.0, 1.0, 4.0, 1.0])
  assert gamma_max == 5.0 and not selected and t == 18 and gamma == _ops.fp32(5.0 * 2.0 ** -18)
  assert G[4, 0].item() == -gamma


def test_gamma_hand_case_selected():
  """Honest values -1, 2, 3, 4, 5, two Byzantine rows, f = 2 (Krum adds 3 distances): mu > 0, R = (12, 6, 4, 4, 6), gamma_max = 4 / 2 + 5
  = 7. The Byzantine score 0 + (1 - g)^2 + (2 + g)^2 first drops below the best honest score 1 + 1 + 4 = 6 (rows 3 and 4) at g = 7 / 32:
  0.78125^2 + 2.21875^2 = 5.533203125, where g = 7 / 16 gives 6.2578125."""
  G = torch.tensor([[-1.0], [2.0], [3.0], [4.0], [5.0], [0.0], [0.0]])
  gamma, selected, t, gamma_max, *_ = _ops.torch_craft_byzantine_(G, [5, 6], "fang-krum", f=2, return_details=True)
  assert gamma_max == 7.0 and selected and t == 5 and gamma == 7.0 / 32
  assert G[5, 0].item() == G[6, 0].item() == -7.0 / 32


def test_degenerate_sums_give_gamma_zero():
  G = torch.randn(6, 40, generator=torch.Generator().manual_seed(2))
  assert _ops.fang_krum_gamma([1.0] * 4, [0.0] * 4, 0.0, [1.0] * 6, 6, 1, [4, 5], 1e-5) == (0.0, False, -1, 0.0)   # C == 0
  G[1, 3] = float("inf")
  gamma, selected, t, gamma_max, *_ = _ops.torch_craft_byzantine_(G, [4, 5], "fang-krum", f=1, return_details=True)
  assert (gamma, selected, t, gamma_max) == (0.0, False, -1, 0.0)
  assert torch.equal(G[4], torch.neg(torch.tensor(0.0)) * _ops._sign(_ops._honest_mean([G[i] for i in range(4)], _ops._scalar(G))))


def test_the_threshold_bounds_the_candidates():
  G = torch.tensor([[1.0], [2.0], [3.0], [4.0], [9.0]])
  for threshold, last in ((1.0, 2), (4.0, 0), (100.0, 0)):   # 5 * 2^-2 = 1.25 >= 1 > 0.625; the first candidate is always tested
    _, selected, t, *_ = _ops.torch_craft_byzantine_(G.clone(), [4], "fang-krum", f=1, threshold=threshold, return_details=True)
    assert not selected and t == last


# ---------------------------------------------------------------------------- #
# fang-trim

def _trim_matrix(n, d, seed, non_finite=False):
  gen = torch.Generator().manual_seed(seed)
  G = torch.randn(1, d, generator=gen) * 0.3 + torch.randn(n, d, generator=gen)
  G[:, ::17] = 0.0   # zero means
  G[0, 5::19] = -0.0
  if non_finite:
    G[0, 3::23] = float("nan")
    G[1, 4::29] = float("inf")
    G[2, 6::31] = float("-inf")
    G[1, 7::37] = float("inf")
    G[2, 7::37] = float("-inf")
  return G


def _python_trim(G, slots, k, beta, key):
  """Per-coordinate pure-Python transcription of fang-trim, in numpy fp32 scalars (one rounding per operation)."""
  n, d = G.shape
  honest = [i for i in range(n) if i not in slots]
  beta = np.float32(beta)
  out = []
  with np.errstate(all="ignore"):
    for x in range(d):
      h = [np.float32(G[i, x].item()) for i in honest]
      mu = h[0]
      for v in h[1:]:
        mu = np.float32(mu + v)
      mu = np.float32(mu / np.float32(len(h)))
      if not (mu > 0 or mu < 0):
        out.append(mu)
        continue
      e = h[0]
      for v in h[1:]:
        if (v < e) if mu > 0 else (v > e):
          e = v
      if mu > 0:
        lo, hi = (np.float32(e * beta), e) if e <= 0 else (np.float32(e / beta), e)
      else:
        lo, hi = (e, np.float32(e * beta)) if e >= 0 else (e, np.float32(e / beta))
      u = np.float32((_ops._splitmix64_int(key ^ (x * 32 + k)) >> 40) * 2.0 ** -24)
      out.append(np.float32(lo + np.float32(u * np.float32(hi - lo))))
  return torch.from_numpy(np.array(out, dtype=np.float32))


@pytest.mark.parametrize("non_finite", [False, True])
@pytest.mark.parametrize("beta", [2.0, 3.5])
def test_trim_reference_matches_a_per_coordinate_transcription(beta, non_finite):
  G = _trim_matrix(7, 301, seed=4, non_finite=non_finite)
  slots = [0, 6] if non_finite else [5, 6]
  key = _ops.fang_trim_key(11, 3)
  crafted = _ops.torch_craft_byzantine_(G.clone(), slots, "fang-trim", scale=beta, seed=11, step=3)
  for k in slots:
    _equal_values(crafted[k], _python_trim(G, slots, k, beta, key))
    _equal_values(crafted[k], _ops.torch_fang_trim_row(G, slots, k, beta, key))
  honest = [i for i in range(7) if i not in slots]
  assert torch.equal(_bits(crafted[honest]), _bits(G[honest]))


def test_trim_values_lie_in_their_interval_past_every_honest_value():
  G = _trim_matrix(9, 2000, seed=5)
  slots = [6, 7, 8]
  crafted = _ops.torch_craft_byzantine_(G.clone(), slots, "fang-trim", step=1)   # beta = 2
  H = G[:6]
  mu = _ops._honest_mean(list(H), _ops._scalar(G))
  low, high = H.min(dim=0).values, H.max(dim=0).values
  pos, neg = mu > 0, mu < 0
  for k in slots:
    b = crafted[k]
    lo = torch.where(low <= 0, low * 2, low / 2)
    assert bool((b[pos] >= lo[pos]).all() and (b[pos] <= low[pos]).all())   # below every honest value
    hi = torch.where(high >= 0, high * 2, high / 2)
    assert bool((b[neg] <= hi[neg]).all() and (b[neg] >= high[neg]).all())   # above every honest value
    zero = ~(pos | neg)
    assert torch.equal(_bits(b[zero]), _bits(mu[zero]))
  assert not torch.equal(crafted[6], crafted[7]) and not torch.equal(crafted[7], crafted[8])


def test_trim_draws_are_keyed_by_seed_and_step():
  G = _trim_matrix(6, 500, seed=6)
  craft = lambda seed, step: _ops.torch_craft_byzantine_(G.clone(), [4, 5], "fang-trim", seed=seed, step=step)
  a, b = craft(0, 1), craft(0, 1)
  assert torch.equal(_bits(a), _bits(b))
  assert not torch.equal(a[4], craft(0, 2)[4]) and not torch.equal(a[4], craft(1, 1)[4])
  u = _ops.fang_trim_uniform(1000, 3, _ops.fang_trim_key(0, 1))
  assert u.dtype == torch.float32 and bool((u >= 0).all() and (u < 1).all()) and 0.4 < float(u.mean()) < 0.6


def test_trim_key_differs_from_bucketing():
  assert _ops.FANG_TAG >= 8 and _ops.FANG_TAG != _ops.BUCKETING_TAG
  key = _ops._splitmix64_int(_ops._splitmix64_int(_ops._splitmix64_int(3) ^ 9) ^ _ops.BUCKETING_TAG)
  assert _ops.fang_trim_key(3, 9) != key


# ---------------------------------------------------------------------------- #
# Arguments

def test_attack_objects():
  attack = attacks.instantiate("fang-krum", 8, 2, [])
  assert attack.omniscient and attack.mode == "fang-krum" and attack.coef is None and attack.threshold == _ops.fp32(1e-5)
  assert attacks.instantiate("fang-krum", 8, 2, ["threshold:0.5"]).threshold == 0.5
  attack = attacks.instantiate("fang-trim", 8, 2, ["scale:3", "seed:42"])
  assert attack.mode == "fang-trim" and attack.scale == 3.0 and attack.seed == 42 and attack.threshold is None
  assert attacks.instantiate("fang-trim", 8, 2, []).scale == 2.0 and attacks.instantiate("fang-trim", 8, 7, []).seed == 0


@pytest.mark.parametrize("mode,n,k,args", [
  ("fang-krum", 8, 2, ["threshold:0"]), ("fang-krum", 8, 2, ["threshold:-1"]), ("fang-krum", 8, 2, ["threshold:inf"]),
  ("fang-krum", 8, 2, ["scale:2"]), ("fang-krum", 5, 2, []), ("fang-krum", 5, 4, []),
  ("fang-trim", 8, 2, ["scale:1"]), ("fang-trim", 8, 2, ["scale:0.5"]), ("fang-trim", 8, 2, ["scale:nan"]), ("fang-trim", 8, 2, ["seed:-1"]),
  ("fang-trim", 8, 2, ["seed:1.5"]), ("fang-trim", 8, 2, ["threshold:1"]), ("fang-trim", 8, 8, [])])
def test_argument_errors(mode, n, k, args):
  with pytest.raises(tools.UserException):
    attacks.instantiate(mode, n, k, args)


def test_reference_rejects_bad_arguments():
  G = torch.randn(6, 10)
  with pytest.raises(tools.UserException):
    _ops.torch_craft_byzantine_(G, [5], "fang-krum")   # f is required
  for f, slots in ((4, [5]), (1, [3, 4, 5]), (True, [5])):   # n - f - 2 = 0; n - 2K - 1 = -1; not an integer
    with pytest.raises(tools.UserException):
      _ops.torch_craft_byzantine_(G, slots, "fang-krum", f=f)
  with pytest.raises(tools.UserException):
    _ops.torch_craft_byzantine_(G, [5], "fang-krum", f=1, threshold=float("nan"))
  with pytest.raises(tools.UserException):
    _ops.torch_craft_byzantine_(G, [5], "fang-trim", seed=0)   # the step key is required
  with pytest.raises(tools.UserException):
    _ops.torch_craft_byzantine_(G, [5], "fang-trim", step=1, scale=1.0)
  with pytest.raises(tools.UserException):
    _ops.torch_craft_byzantine_(G, [5], "fang-trim", step=1, return_details=True)
  with pytest.raises(tools.UserException):
    gar_ops.craft_byzantine_(G, [5], "fang-krum", f=1, threshold=0.0)
  out = gar_ops.craft_byzantine_(G.clone(), [4, 5], "fang-krum", f=1, return_details=True)   # CPU rows: the reference
  assert out == _ops.torch_craft_byzantine_(G.clone(), [4, 5], "fang-krum", f=1, return_details=True)


# ---------------------------------------------------------------------------- #
# Host engine end to end

@pytest.mark.parametrize("rule", ["krum", "trimmed-mean", "median"])
@pytest.mark.parametrize("mode", ["fang-krum", "fang-trim"])
def test_host_engine_trains_with_the_attack(mode, rule):
  n, k = 7, 2
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  attack = attacks.instantiate(mode, n, k, ["seed:5"] if mode == "fang-trim" else [])
  mgr = Manager(experiment, aggregators.instantiate(rule, n, k, []), n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu", attack=attack,
                nb_real_byz=k, seed=1)
  assert mgr.aggregation.name == "host" and mgr.byzantine_slots == [5, 6]
  for _ in range(2):
    loss = float(mgr.train())
    assert math.isfinite(loss)
    rows = mgr.aggregation.visible_rows()
    G = torch.stack([rows[i] for i in range(n)])
    honest = [G[i] for i in range(5)]
    if mode == "fang-krum":
      gamma, selected, t, gamma_max, A, B, C, T = mgr.aggregation.last_craft
      assert (gamma, selected, t, gamma_max) == _ops.fang_krum_gamma(A, B, C, T, n, 2, [5, 6], 1e-5) and gamma > 0
      expected = torch.neg(torch.tensor(gamma)) * _ops._sign(_ops._honest_mean(honest, _ops._scalar(G)))
      assert torch.equal(G[5], expected) and torch.equal(G[6], expected)
    else:   # the step key is the number of the update the rows fed
      key = _ops.fang_trim_key(5, mgr.aggregation.updates)
      for slot in (5, 6):
        _equal_values(G[slot], _ops.torch_fang_trim_row(G, [5, 6], slot, 2.0, key))


# ---------------------------------------------------------------------------- #
# Runner CLI

def _run(args, timeout=300):
  env = dict(os.environ, AGB_NUM_THREADS="2", OMP_NUM_THREADS="2")
  proc = subprocess.run([sys.executable, str(ROOT / "runner.py")] + args, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=timeout, env=env, cwd=str(ROOT))
  return proc.returncode, proc.stdout.decode(errors="replace")


@pytest.mark.parametrize("attack", [["--attack", "fang-krum", "--attack-args", "threshold:1e-4"], ["--attack", "fang-trim", "--attack-args", "scale:3"]])
def test_runner_accepts_the_attacks(attack):
  args = LOCAL + ["--experiment", "mnist", "--aggregator", "krum", "--nb-workers", "7", "--nb-decl-byz-workers", "2", "--nb-real-byz-workers", "2",
                  "--max-step", "3", "--seed", "3", "--learning-rate-args", "initial-rate:0.05", "--evaluation-file", "-", "--summary-dir", "-",
                  "--evaluation-delta", "1000", "--evaluation-period", "-1", "--checkpoint-period", "-1", "--checkpoint-delta", "1000"] + attack
  code, out = _run(args)
  assert code == 0, out
  losses = re.findall(r"Step \d+: total loss = ([0-9.eE+-]+|NaN)", out)
  assert len(losses) == 3 and all(math.isfinite(float(x)) for x in losses), out
  code, out = _run(args[:-1] + ["bogus:1"])
  assert code != 0 and "bogus" in out

"""Min-Max and Min-Sum (Shejwalkar & Houmansadr, NDSS 2021) on the CPU: the torch reference against exact hand cases and an independent
float64 transcription of the authors' search, the tightness of the constraint, the argument checks, the host engine end to end and the
runner CLI."""

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
MODES = ("min-max", "min-sum")
DEVIATIONS = ("unit-vec", "sign", "std")


def _fp32(x):
  return float(np.float32(x))


def _bits(t):
  return t.detach().cpu().contiguous().view(torch.int32)


def _craft(G, byz, mode, deviation):
  """(crafted copy of G, (gamma, A, B, C, T))"""
  out = G.clone()
  details = _ops.torch_craft_byzantine_(out, byz, mode, None, deviation=deviation, return_details=True)
  return out, details


# ---------------------------------------------------------------------------- #
# Exact hand cases

@pytest.mark.parametrize("deviation", ["unit-vec", "sign"])
def test_hand_case_two_honest_rows(deviation):
  """h = (0, 0), (2, 0): mu = (1, 0) = p (unit-vec and sign), A = (1, 1), B = (1, -1), C = 1, T = 4. Min-Max: gamma_1 = (1 + 2) / 1,
  gamma_2 = 3 / (2 + 1) = 1; Min-Sum: sqrt(1 / 1) = 1. Both give b = (0, 0): ||b - h_2||^2 = 4 = T, and 0 + 4 = max_i sum_j D_ij."""
  G = torch.tensor([[0.0, 0.0], [2.0, 0.0], [7.0, -7.0]])
  for mode in MODES:
    out, (gamma, A, B, C, T) = _craft(G, [2], mode, deviation)
    assert (gamma, A, B, C) == (1.0, [1.0, 1.0], [1.0, -1.0], 1.0)
    assert T == (4.0 if mode == "min-max" else None)
    assert out[2].tolist() == [0.0, 0.0] and torch.equal(out[:2], G[:2])


def test_hand_case_three_honest_rows():
  """h = (0, 0), (3, 0), (0, 3), Byzantine slot first: mu = p = (1, 1), A = (2, 5, 5), B = (2, -1, -1), C = 2, T = 18.
  Min-Max: gamma = min(4, 13 / (sqrt(27) + 1)) = (sqrt(27) - 1) / 2, the root of ||b - h_2||^2 = 2 g^2 + 2 g + 5 = 18.
  Min-Sum: 12 + 6 g^2 = 27 (the largest row sum of distances, 9 + 18), g = sqrt(5 / 2)."""
  G = torch.tensor([[9.0, 9.0], [0.0, 0.0], [3.0, 0.0], [0.0, 3.0]])
  out, (gamma, A, B, C, T) = _craft(G, [0], "min-max", "unit-vec")
  assert (A, B, C, T) == ([2.0, 5.0, 5.0], [2.0, -1.0, -1.0], 2.0, 18.0)
  assert gamma == _fp32(13.0 / (math.sqrt(27.0) + 1.0)) and abs(gamma - (math.sqrt(27.0) - 1.0) / 2.0) < 1e-6
  assert out[0].tolist() == [_fp32(1.0 - gamma)] * 2
  out, (gamma, A, B, C, T) = _craft(G, [0], "min-sum", "unit-vec")
  assert gamma == _fp32(math.sqrt(2.5)) and T is None
  assert out[0].tolist() == [_fp32(1.0 - gamma)] * 2


def test_sign_with_zeros_in_the_mean():
  """sign(mu) is +1, -1, +0 for +0 and -0, NaN for NaN; b = mu - gamma * p keeps mu where p = 0 (a -0 mean stays -0)."""
  G = torch.tensor([[1.0, -1.0, 3.0, -0.0, -2.0],
                    [-1.0, 1.0, 1.0, -0.0, -4.0],
                    [0.0, 0.0, 0.0, 0.0, 0.0]])
  mu, p = _ops.optimized_deviation(G, [2], "min-max", "sign")
  assert mu.tolist() == [0.0, 0.0, 2.0, 0.0, -3.0]
  assert _bits(p).tolist() == _bits(torch.tensor([0.0, 0.0, 1.0, 0.0, -1.0])).tolist()   # +0, never -0
  for mode in MODES:
    out, (gamma, *_) = _craft(G, [2], mode, "sign")
    assert gamma > 0
    assert _bits(out[2, :2]).tolist() == [0, 0] and _bits(out[2, 3:4]).tolist() == _bits(torch.tensor([-0.0])).tolist()
    assert out[2, 2].item() == _fp32(2.0 - gamma) and out[2, 4].item() == _fp32(-3.0 + gamma)


def test_unit_vec_with_a_zero_mean_gives_gamma_zero():
  G = torch.tensor([[1.0, 2.0, -3.0], [-1.0, -2.0, 3.0], [5.0, 5.0, 5.0]])
  for mode in MODES:
    out, (gamma, A, B, C, T) = _craft(G, [2], mode, "unit-vec")
    assert C == 0.0 and gamma == 0.0
    assert out[2].tolist() == [0.0, 0.0, 0.0]


def test_identical_honest_rows_under_std_give_the_mean():
  G = torch.tensor([[0.5, -1.25, 3.0]] * 3 + [[9.0, 9.0, 9.0]])
  for mode in MODES:
    out, (gamma, A, B, C, T) = _craft(G, [3], mode, "std")
    assert C == 0.0 and gamma == 0.0 and A == [0.0] * 3
    assert torch.equal(out[3], G[0])


@pytest.mark.parametrize("deviation", DEVIATIONS)
@pytest.mark.parametrize("mode", MODES)
def test_non_finite_honest_values_give_gamma_zero(mode, deviation):
  """A NaN or infinite honest value makes the sums non-finite: gamma = 0, and b = mu - 0 * p follows IEEE arithmetic."""
  G = torch.randn(6, 40, generator=torch.Generator().manual_seed(5))
  G[0, 3] = float("nan")
  G[1, 7] = float("inf")
  out, (gamma, *_) = _craft(G, [4, 5], mode, deviation)
  assert gamma == 0.0
  mu, p = _ops.optimized_deviation(G, [4, 5], mode, deviation)
  expected = mu - torch.tensor(0.0) * p
  for i in (4, 5):
    assert torch.equal(torch.isnan(out[i]), torch.isnan(expected))
    finite = ~torch.isnan(expected)
    assert torch.equal(out[i][finite], expected[finite])
  assert math.isnan(out[4, 3].item())
  if deviation == "sign":
    assert out[4, 7].item() == math.inf   # p = +1 there, inf - 0 * 1 = inf
  else:
    assert math.isnan(out[4, 7].item())   # unit-vec: 0 * inf; std: sigma = NaN (inf - inf)
  finite_cols = [c for c in range(40) if c not in (3, 7)]
  assert torch.equal(out[4, finite_cols], mu[finite_cols])


# ---------------------------------------------------------------------------- #
# Independent float64 oracle: the authors' halving search on explicit distances

def _authors_search(H, b_of, mode):
  """Shejwalkar & Houmansadr's search for the coefficient (their `lamda`, started at 10 with a halving step: it brackets the root
  below 20), on explicit float64 distances; run to 1e-13 instead of their 1e-5."""
  dist = ((H[:, None, :] - H[None, :, :]) ** 2).sum(axis=2)
  bound = dist.max() if mode == "min-max" else dist.sum(axis=1).max()

  def feasible(lam):
    d = ((b_of(lam)[None, :] - H) ** 2).sum(axis=1)
    return (d.max() if mode == "min-max" else d.sum()) <= bound

  lam, step, succ = 10.0, 10.0, 0.0
  while abs(succ - lam) > 1e-13:
    if feasible(lam):
      succ = lam
      lam = lam + step / 2
    else:
      lam = lam - step / 2
    step = step / 2
  return succ


def _oracle_deviation(H, deviation):
  mu = H.mean(axis=0)
  if deviation == "unit-vec":
    return mu, mu / np.linalg.norm(mu)
  if deviation == "sign":
    return mu, np.sign(mu)
  return mu, H.std(axis=0, ddof=1)


def _oracle_cases():
  rng = np.random.default_rng(2021)
  for n in range(3, 41):
    for deviation in DEVIATIONS:
      k = int(rng.integers(1, n - 1))
      yield n, k, deviation, int(rng.integers(0, 2 ** 31))


@pytest.mark.parametrize("mode", MODES)
def test_gamma_matches_the_authors_search_in_float64(mode):
  checked = 0
  for n, k, deviation, seed in _oracle_cases():
    rng = np.random.default_rng(seed)
    d = 64
    G = torch.tensor(rng.normal(0.0, 1.0, (1, d)) + rng.normal(0.0, 0.3, (n, d)), dtype=torch.float32)
    byz = sorted(rng.choice(n, size=k, replace=False).tolist())
    _, (gamma, A, B, C, T) = _craft(G, byz, mode, deviation)
    H = G[[i for i in range(n) if i not in byz]].double().numpy()
    mu, p = _oracle_deviation(H, deviation)
    coef = _ops.optimized_coefficient(deviation, gamma, C)   # unit-vec: the push along mu / ||mu||
    if coef >= 19.0:
      continue   # outside the search's bracket
    lam = _authors_search(H, lambda lam: mu - lam * p, mode)
    assert abs(coef - lam) <= 1e-5 * lam, (n, k, deviation, coef, lam)
    checked += 1
  assert checked >= 100


@pytest.mark.parametrize("deviation", DEVIATIONS)
@pytest.mark.parametrize("mode", MODES)
def test_the_crafted_row_meets_its_constraint_tightly(mode, deviation):
  """In float64, from the crafted fp32 row: Min-Max's max_i ||b - h_i||^2 and Min-Sum's sum_i ||b - h_i||^2 lie in
  [bound (1 - 1e-4), bound (1 + 1e-5)]."""
  for seed in range(12):
    rng = np.random.default_rng(100 + seed)
    n = int(rng.integers(3, 33))
    k = int(rng.integers(1, n - 1))
    G = torch.tensor(rng.normal(0.0, 1.0, (1, 500)) + rng.normal(0.0, 0.5, (n, 500)), dtype=torch.float32)
    out, (gamma, *_) = _craft(G, list(range(n - k, n)), mode, deviation)
    H = G[:n - k].double().numpy()
    b = out[n - 1].double().numpy()
    dist = ((H[:, None, :] - H[None, :, :]) ** 2).sum(axis=2)
    bound = dist.max() if mode == "min-max" else dist.sum(axis=1).max()
    d = ((b[None, :] - H) ** 2).sum(axis=1)
    value = d.max() if mode == "min-max" else d.sum()
    assert gamma > 0 and bound * (1 - 1e-4) <= value <= bound * (1 + 1e-5), (n, k, value, bound)


def test_gamma_solver_matches_the_closed_forms():
  A, B, C, T = [2.0, 5.0, 5.0], [2.0, -1.0, -1.0], 2.0, 18.0
  assert _ops.optimized_gamma("min-max", A, B, C, T) == _fp32(13.0 / (math.sqrt(27.0) + 1.0))
  assert _ops.optimized_gamma("min-sum", A, B, C) == _fp32(math.sqrt(2.5))
  assert _ops.optimized_gamma("min-max", A, B, 0.0, T) == 0.0
  assert _ops.optimized_gamma("min-max", A, B, C, math.inf) == 0.0
  assert _ops.optimized_gamma("min-sum", [math.nan] + A[1:], B, C) == 0.0


def test_ops_front_end_falls_back_to_the_reference_on_cpu():
  G = torch.randn(7, 333, generator=torch.Generator().manual_seed(3))
  expected, details = _craft(G, [5, 6], "min-max", "std")
  out = G.clone()
  assert gar_ops.craft_byzantine_(out, [5, 6], "min-max", deviation="std", return_details=True) == details
  assert torch.equal(out, expected)
  row = _ops.torch_optimized_row(G, [5, 6], "min-max", "std", details[0])
  assert torch.equal(expected[5], row) and torch.equal(expected[6], row)


# ---------------------------------------------------------------------------- #
# Arguments

@pytest.mark.parametrize("mode", MODES)
def test_attack_objects(mode):
  attack = attacks.instantiate(mode, 8, 2, [])
  assert attack.omniscient and attack.mode == mode and attack.deviation == "unit-vec" and attack.coef is None
  assert attacks.instantiate(mode, 8, 2, ["deviation:std"]).deviation == "std"
  assert attacks.instantiate("alie", 8, 2, []).deviation is None and attacks.instantiate("ipm", 8, 2, []).deviation is None
  assert attacks.instantiate(mode, 3, 1, []).deviation == "unit-vec"   # H = 2 is enough


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("n,k,args", [(8, 2, ["deviation:median"]), (8, 2, ["z:1.0"]), (3, 2, []), (8, 0, []), (8, 8, [])])
def test_argument_errors(mode, n, k, args):
  with pytest.raises(tools.UserException):
    attacks.instantiate(mode, n, k, args)


def test_reference_rejects_bad_arguments():
  G = torch.randn(4, 8)
  with pytest.raises(tools.UserException, match="deviation"):
    _ops.torch_craft_byzantine_(G, [3], "min-max", None, deviation="l2")
  with pytest.raises(tools.UserException, match="honest"):
    _ops.torch_craft_byzantine_(G, [1, 2, 3], "min-sum", None)
  with pytest.raises(tools.UserException):
    _ops.torch_craft_byzantine_(G, [], "min-max", None)
  with pytest.raises(tools.UserException, match="return_details"):
    _ops.torch_craft_byzantine_(G, [3], "alie", 1.0, return_details=True)


@pytest.mark.parametrize("mode", MODES)
def test_authentication_is_refused(mode):
  experiment = experiments.instantiate("mnist", ["batch-size:8"])
  gar = aggregators.instantiate("average", 5, 2, [])
  with pytest.raises(tools.UserException, match="authenticate"):
    Manager(experiment, gar, 5, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu", attack=attacks.instantiate(mode, 5, 2, []), nb_real_byz=2,
            authenticate=True)


# ---------------------------------------------------------------------------- #
# Host engine end to end

@pytest.mark.parametrize("deviation", DEVIATIONS)
@pytest.mark.parametrize("mode", MODES)
def test_host_engine_trains_with_the_attack(mode, deviation):
  n, k = 6, 2
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  attack = attacks.instantiate(mode, n, k, ["deviation:" + deviation])
  mgr = Manager(experiment, aggregators.instantiate("median", n, k, []), n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu", attack=attack,
                nb_real_byz=k, seed=1)
  assert mgr.aggregation.name == "host" and mgr.byzantine_slots == [4, 5]
  for _ in range(2):
    loss = float(mgr.train())
    assert math.isfinite(loss)
    rows = mgr.aggregation.visible_rows()
    G = torch.stack([rows[i] for i in range(n)])
    gamma, A, B, C, T = mgr.aggregation.last_craft
    assert gamma > 0 and gamma == _ops.optimized_gamma(mode, A, B, C, T)
    expected = _ops.torch_optimized_row(G, [4, 5], mode, deviation, gamma)
    assert torch.equal(G[4], expected) and torch.equal(G[5], expected)


# ---------------------------------------------------------------------------- #
# Runner CLI

def _run(args, timeout=300):
  env = dict(os.environ, AGB_NUM_THREADS="2", OMP_NUM_THREADS="2")
  proc = subprocess.run([sys.executable, str(ROOT / "runner.py")] + args, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=timeout, env=env, cwd=str(ROOT))
  return proc.returncode, proc.stdout.decode(errors="replace")


@pytest.mark.parametrize("attack", [["--attack", "min-max", "--attack-args", "deviation:std"], ["--attack", "min-sum"]])
def test_runner_accepts_the_attacks(attack):
  args = LOCAL + ["--experiment", "mnist", "--aggregator", "krum", "--nb-workers", "7", "--nb-decl-byz-workers", "2", "--nb-real-byz-workers", "2",
                  "--max-step", "3", "--seed", "3", "--learning-rate-args", "initial-rate:0.05", "--evaluation-file", "-", "--summary-dir", "-",
                  "--evaluation-delta", "1000", "--evaluation-period", "-1", "--checkpoint-period", "-1", "--checkpoint-delta", "1000"] + attack
  code, out = _run(args)
  assert code == 0, out
  losses = re.findall(r"Step \d+: total loss = ([0-9.eE+-]+|NaN)", out)
  assert len(losses) == 3 and all(math.isfinite(float(x)) for x in losses), out
  code, out = _run(args[:-1] + ["deviation:l1"] if attack[-1].startswith("deviation") else args + ["--attack-args", "deviation:l1"])
  assert code != 0 and "deviation" in out

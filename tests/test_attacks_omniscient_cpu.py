"""Omniscient attacks (ALIE, IPM) on the CPU: the torch reference against exact hand cases and a float64 oracle, the default z, the
argument checks, the host engine end to end, ALIE steering Krum, and the runner CLI."""

import math
import os
import pathlib
import re
import subprocess
import sys

import numpy as np
import pytest
import scipy.stats
import torch

from aggregathor_b200 import aggregators, attacks, experiments, tools
from aggregathor_b200.aggregators import _ops
from aggregathor_b200.engine.trainer import Manager
from aggregathor_b200.ops import gar as gar_ops

ROOT = pathlib.Path(__file__).resolve().parent.parent
LOCAL = ["--server", '{"local": ["127.0.0.1:7000"]}', "--ps-job-name", "local", "--wk-job-name", "local", "--ev-job-name", "local", "--no-wait"]
U = 2.0 ** -24   # unit roundoff of fp32


def _run(args, timeout=300):
  env = dict(os.environ, AGB_NUM_THREADS="2", OMP_NUM_THREADS="2")
  proc = subprocess.run([sys.executable, str(ROOT / "runner.py")] + args, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=timeout, env=env, cwd=str(ROOT))
  return proc.returncode, proc.stdout.decode(errors="replace")


def _craft(G, byz, mode, coef):
  return _ops.torch_craft_byzantine_(G.clone(), byz, mode, coef)


# ---------------------------------------------------------------------------- #
# Exact hand cases

def test_hand_case_mean_two_sigma_two():
  G = torch.tensor([[0.0, -4.0], [2.0, -2.0], [4.0, 0.0], [123.0, 7.0]])
  # honest {0, 2, 4}: mu = 2, v = (4 + 0 + 4) / 2 = 4, sigma = 2
  out = _craft(G, [3], "alie", 0.5)
  assert out[3].tolist() == [3.0, -1.0]
  assert torch.equal(out[:3], G[:3])
  out = _craft(G, [3], "ipm", 0.5)
  assert out[3].tolist() == [-1.0, 1.0]


def test_hand_case_two_honest_rows():
  # H = 2: mu = 3, v = ((1 - 3)^2 + (5 - 3)^2) / 1 = 8, sigma = sqrt(8); z = sqrt(2) rounded to fp32 is not exact, so use z = 0.25
  G = torch.tensor([[1.0], [5.0], [0.0], [0.0]])
  out = _craft(G, [2, 3], "alie", 0.25)
  expected = np.float32(3.0) + np.float32(0.25) * np.sqrt(np.float32(8.0))
  assert out[2].item() == out[3].item() == float(np.float32(expected))
  assert _craft(G, [2, 3], "ipm", 2.0)[2:].flatten().tolist() == [-6.0, -6.0]


def test_hand_case_single_coordinate_and_slot_positions():
  # a single coordinate; the Byzantine slots need not be the last ones
  G = torch.tensor([[10.0], [4.0], [-3.0], [2.0], [0.0]])
  out = _craft(G, [1, 2], "alie", 1.0)   # honest 10, 2, 0: mu = 4, v = (36 + 4 + 16) / 2 = 28
  assert out[1].item() == out[2].item() == float(np.float32(4.0) + np.sqrt(np.float32(28.0)))
  assert [out[i].item() for i in (0, 3, 4)] == [10.0, 2.0, 0.0]


@pytest.mark.parametrize("n", [3, 5, 9])
def test_k_one_and_k_n_minus_two(n):
  gen = torch.Generator().manual_seed(n)
  G = torch.randint(-8, 9, (n, 17), generator=gen).float()
  for byz in ([n - 1], list(range(2, n))):
    honest = G[[i for i in range(n) if i not in byz]].double()
    # small integers: the mean of H values is exact up to one division, which the fp32 path rounds the same way
    mu = honest.sum(0) / honest.shape[0]
    out = _craft(G, byz, "ipm", 1.0)
    assert torch.equal(out[byz[0]], (-mu).float())
    out = _craft(G, byz, "alie", 0.0)
    assert torch.equal(out[byz[-1]], mu.float())
    assert all(torch.equal(out[i], out[byz[0]]) for i in byz)


@pytest.mark.parametrize("H", [2, 7, 8, 9, 30])
def test_reference_rounds_every_operation_once(H):
  """The torch reference equals a step-by-step fp32 NumPy evaluation of the definition bit for bit (NumPy's fp32 add, multiply,
  divide and square root are the correctly rounded IEEE operations)."""
  n, d = H + 2, 20011
  G = torch.randn(n, d, generator=torch.Generator().manual_seed(H)) * torch.logspace(-3, 3, d)
  h = G[:H].numpy()
  f32 = np.float32
  mu = h[0].copy()
  for i in range(1, H):
    mu = mu + h[i]
  mu = mu / f32(H)
  var = np.zeros(d, dtype=f32)
  for i in range(H):
    dev = h[i] - mu
    var = dev * dev if i == 0 else var + dev * dev
  z, eps = f32(0.75), f32(0.1)
  alie = mu + z * np.sqrt(var / f32(H - 1))
  ipm = -eps * mu
  assert alie.dtype == ipm.dtype == np.float32
  assert np.array_equal(_ops.torch_byzantine_row(G, [H, H + 1], "alie", float(z)).numpy().view(np.int32), alie.view(np.int32))
  assert np.array_equal(_ops.torch_byzantine_row(G, [H, H + 1], "ipm", float(eps)).numpy().view(np.int32), ipm.view(np.int32))


def test_non_finite_values_propagate():
  G = torch.tensor([[1.0, float("nan"), float("inf"), 1.0], [2.0, 0.0, 1.0, float("inf")], [3.0, 1.0, 2.0, float("-inf")], [0.0, 0.0, 0.0, 0.0]])
  out = _craft(G, [3], "alie", 1.0)
  assert out[3, 0].item() == 3.0 and all(math.isnan(v) for v in out[3, 1:].tolist())
  out = _craft(G, [3], "ipm", 1.0)
  assert out[3, 0].item() == -2.0 and math.isnan(out[3, 1].item()) and out[3, 2].item() == -math.inf and math.isnan(out[3, 3].item())


# ---------------------------------------------------------------------------- #
# Against a float64 oracle

def _oracle(G, byz, mode, coef):
  honest = np.stack([G[i].numpy().astype(np.float64) for i in range(G.shape[0]) if i not in byz])
  mu = honest.mean(axis=0)
  if mode == "ipm":
    return -coef * mu
  return mu + coef * np.sqrt(((honest - mu) ** 2).sum(axis=0) / (honest.shape[0] - 1))


def _error_bound(H, M, mode, coef):
  """Forward error bound of the fp32 evaluation, per coordinate, from H and the largest honest magnitude M of the coordinate.
  mu: H - 1 rounded additions of terms <= M in size (error <= (H - 1) u H M), divided by H, plus the rounding of the quotient
  -> err_mu <= H u M (1 + H u). Deviations |h - mu| <= 2 M, each carrying err_mu + 2 u M; the sum of H squares, the division and the
  square root add (H + 3) u relative to ||dev|| <= 2 M sqrt(H); with r = sqrt(H / (H - 1)), err_sigma <= r (err_mu + 2 u M) +
  (H + 3) u r 2 M. The final multiply and add round once each relative to |b| <= M + |z| 2 r M."""
  err_mu = H * U * M * (1 + H * U)
  if mode == "ipm":
    return abs(coef) * err_mu + U * abs(coef) * M
  r = math.sqrt(H / (H - 1))
  err_sigma = r * (err_mu + 2 * U * M) + (H + 3) * U * r * 2 * M
  return err_mu + abs(coef) * (err_sigma + U * 2 * r * M) + 2 * U * (M + abs(coef) * 2 * r * M)


@pytest.mark.parametrize("mode", ["alie", "ipm"])
@pytest.mark.parametrize("n", list(range(3, 41)))
def test_reference_matches_float64_oracle(n, mode):
  gen = torch.Generator().manual_seed(1000 + n)
  G = torch.randn(n, 2048, generator=gen) * torch.logspace(-3, 3, 2048)   # magnitudes spread over six decades
  k = max(1, n // 4)
  byz = list(range(n - k, n))
  coef = attacks.instantiate(mode, n, k, []).coef if mode == "ipm" or k <= n // 2 else 1.5
  out = _craft(G, byz, mode, coef)
  ref = _oracle(G, byz, mode, coef)
  H = n - k
  M = G[:n - k].abs().amax(dim=0).double().numpy()
  bound = _error_bound(H, M, mode, coef)
  assert np.all(bound < 1e-4 * M)   # the bound is meaningful: far below the values themselves
  err = np.abs(out[n - k].double().numpy() - ref)
  assert np.all(err <= bound), (float((err / bound).max()), int((err / bound).argmax()))
  assert torch.equal(out[:n - k], G[:n - k])


def test_ops_front_end_falls_back_to_the_reference_on_cpu():
  G = torch.randn(6, 1001, generator=torch.Generator().manual_seed(3))
  expected = _craft(G, [4, 5], "alie", 0.7)
  assert torch.equal(gar_ops.craft_byzantine_(G, [4, 5], "alie", 0.7), expected)
  assert torch.equal(G, expected)


# ---------------------------------------------------------------------------- #
# Default z

def test_default_z_reference_values():
  for (n, k), value in {(7, 2): "0.56594884", (8, 2): "0.31863937", (19, 4): "0.47950566", (32, 6): "0.40225005"}.items():
    z = attacks.instantiate("alie", n, k, []).coef
    assert "%.8f" % z == value
    assert z == float(np.float32(z))


def test_default_z_matches_scipy_for_every_valid_configuration():
  checked = 0
  for n in range(3, 33):
    for k in range(1, min(n // 2, n - 2) + 1):
      s = (n // 2 + 1) - k
      expected = float(np.float32(scipy.stats.norm.ppf((n - s) / n)))
      assert attacks.instantiate("alie", n, k, []).coef == expected, (n, k)
      checked += 1
  assert checked > 200


def test_coefficients_are_rounded_to_fp32():
  assert attacks.instantiate("alie", 8, 2, ["z:0.1"]).coef == float(np.float32(0.1))
  assert attacks.instantiate("ipm", 8, 2, []).coef == float(np.float32(0.1))
  assert attacks.instantiate("ipm", 8, 2, ["epsilon:3"]).coef == 3.0
  attack = attacks.instantiate("ipm", 8, 2, [])
  assert attack.omniscient and attack.mode == "ipm" and not attacks.instantiate("flip", 8, 2, []).omniscient


# ---------------------------------------------------------------------------- #
# Argument errors

@pytest.mark.parametrize("name,n,k,args", [
  ("alie", 8, 0, []), ("ipm", 8, 0, []), ("alie", 8, 8, ["z:1"]), ("ipm", 8, 8, []),
  ("alie", 8, 7, ["z:1"]),                                  # H = 1 < 2
  ("alie", 8, 2, ["z:inf"]), ("alie", 8, 2, ["z:nan"]), ("alie", 8, 2, ["z:1e39"]), ("alie", 8, 2, ["z:abc"]),
  ("ipm", 8, 2, ["epsilon:nan"]), ("ipm", 8, 2, ["epsilon:-inf"]),
  ("alie", 8, 5, []), ("alie", 7, 4, []),                   # default z needs k <= floor(n / 2)
])
def test_argument_errors(name, n, k, args):
  with pytest.raises(tools.UserException):
    attacks.instantiate(name, n, k, args)


def test_arguments_at_the_bounds_are_accepted():
  assert attacks.instantiate("alie", 8, 4, []).coef == float(np.float32(scipy.stats.norm.ppf(7 / 8)))   # s = 1
  assert attacks.instantiate("alie", 8, 6, ["z:2"]).coef == 2.0   # H = 2
  assert attacks.instantiate("ipm", 8, 7, []).coef > 0            # H = 1


def test_reference_rejects_bad_slots():
  G = torch.zeros(4, 8)
  for byz, mode in (([], "alie"), ([4], "ipm"), ([1, 2, 3], "alie"), ([0, 1, 2, 3], "ipm"), ([1], "nope")):
    with pytest.raises(tools.UserException):
      _ops.torch_craft_byzantine_(G, byz, mode, 1.0)


def test_authentication_is_refused():
  experiment = experiments.instantiate("mnist", ["batch-size:8"])
  gar = aggregators.instantiate("average", 5, 2, [])
  for name in ("alie", "ipm"):
    with pytest.raises(tools.UserException, match="authenticate"):
      Manager(experiment, gar, 5, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu", attack=attacks.instantiate(name, 5, 2, []), nb_real_byz=2,
              authenticate=True)


# ---------------------------------------------------------------------------- #
# Host engine end to end

def _manager(gar_name, n, f, attack=None, real=0, seed=0):
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate(gar_name, n, f, [])
  return Manager(experiment, gar, n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu", attack=attack, nb_real_byz=real, seed=seed)


@pytest.mark.parametrize("mode", ["alie", "ipm"])
def test_host_engine_crafts_the_byzantine_rows(mode):
  n, k = 5, 2
  attack = attacks.instantiate(mode, n, k, [])
  mgr = _manager("average", n, k, attack, k)
  plain = _manager("average", n, k)
  assert mgr.aggregation.name == "host" and mgr.byzantine_slots == [3, 4]
  loss = float(mgr.train())
  plain.train()
  assert math.isfinite(loss)
  rows = mgr.aggregation.visible_rows()
  G = torch.stack([rows[i] for i in range(n)])
  honest_before = torch.stack([plain.aggregation.visible_rows()[i] for i in range(n - k)])
  assert torch.equal(G[:n - k], honest_before)   # honest rows are never written
  expected = _ops.torch_byzantine_row(G, [3, 4], mode, attack.coef)
  assert torch.equal(G[3], expected) and torch.equal(G[4], expected)
  assert not torch.equal(G[3], plain.aggregation.visible_rows()[3])
  # the rule aggregated the crafted matrix: its mean, added in worker order and divided once
  mean = G[0].clone()
  for i in range(1, n):
    mean = mean + G[i]
  assert torch.equal(mgr.aggregation.last_aggregate, mean / torch.tensor(float(n)))


def test_alie_steers_krum():
  """n = 8, k = 2, d = 10^4, Gaussian rows (sigma = 1), z = z_max(8, 2) = 0.3186. Squared distances concentrate around their means:
  honest-honest ~ 2 d sigma^2; Byzantine-honest ~ d sigma^2 (1 + z^2) (b sits at mu + z sigma, h - mu has variance ~ sigma^2);
  Byzantine-Byzantine = 0. Krum (f = 2) sums the n - f - 2 = 4 smallest distances: a Byzantine row scores 0 + 3 d (1 + z^2) ~ 3.3 d,
  an honest row at best 2 d (1 + z^2) + 2 * 2 d ~ 6.2 d. The relative spread of each distance is ~ sqrt(2 / d) ~ 1.4 %, far below
  the gap, so a Byzantine row wins; the two tie exactly and the lower slot (6) is selected. With m = 1 the aggregate is that row."""
  n, k, d = 8, 2, 10 ** 4
  G = torch.randn(n, d, generator=torch.Generator().manual_seed(42))
  attack = attacks.instantiate("alie", n, k, [])
  _ops.torch_craft_byzantine_(G, [6, 7], "alie", attack.coef)
  gar = aggregators.instantiate("krum", n, 2, ["m:1"])
  out = gar.aggregate(G)
  assert torch.equal(out, G[6])
  _, selected = _ops.host_krum(G, 2, 1, return_selected=True)
  assert selected.tolist() == [6]


# ---------------------------------------------------------------------------- #
# Runner CLI

@pytest.mark.parametrize("attack", [["--attack", "alie"], ["--attack", "ipm", "--attack-args", "epsilon:0.5"]])
def test_runner_accepts_omniscient_attacks(attack):
  args = LOCAL + ["--experiment", "mnist", "--aggregator", "median", "--nb-workers", "5", "--nb-decl-byz-workers", "2", "--nb-real-byz-workers", "2",
                  "--max-step", "4", "--seed", "3", "--learning-rate-args", "initial-rate:0.05", "--evaluation-file", "-", "--summary-dir", "-",
                  "--evaluation-delta", "1000", "--evaluation-period", "-1", "--checkpoint-period", "-1", "--checkpoint-delta", "1000"] + attack
  runs = []
  for _ in range(2):
    code, out = _run(args)
    assert code == 0, out
    losses = re.findall(r"Step \d+: total loss = ([0-9.eE+-]+|NaN)", out)
    assert len(losses) == 4 and all(math.isfinite(float(x)) for x in losses), out
    runs.append(losses)
  assert runs[0] == runs[1]

"""DnC on the host: the sampler, the scores against the paper's SVD definition, the Jacobi against LAPACK, hand cases, Min-Max rows,
the host library against the torch reference, argument checks, the host engine and checkpoint / resume through the runner."""

import math
import os
import pathlib
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from aggregathor_b200 import aggregators, tools
from aggregathor_b200.aggregators import FusedSpec, _ops
from aggregathor_b200.engine.flat import FlatLayout
from aggregathor_b200.engine.optimizers import optimizers
from aggregathor_b200.engine.schedules import build
from aggregathor_b200.parallel.aggregation import HostAggregation

ROOT = pathlib.Path(__file__).resolve().parent.parent
LOCAL = ["--server", '{"local": ["127.0.0.1:7000"]}', "--ps-job-name", "local", "--wk-job-name", "local", "--ev-job-name", "local", "--no-wait"]


# ---------------------------------------------------------------------------- #
# Sampler

@pytest.mark.parametrize("domain", [1, 2, 3, 5, 64, 1000, 65537, 25557032])
def test_sampler_draws_distinct_coordinates_in_range(domain):
  s = _ops.dnc_sample(domain, 10000, seed=3, step=7, t=1)
  assert s.dtype == np.int64 and len(s) == min(10000, domain)
  assert len(np.unique(s)) == len(s) and s.min() >= 0 and s.max() < domain
  assert np.array_equal(s, _ops.dnc_sample(domain, 10000, seed=3, step=7, t=1))
  if domain <= 10000:
    assert np.array_equal(np.sort(s), np.arange(domain))


def test_sampler_changes_with_seed_step_and_iteration():
  base = _ops.dnc_sample(1 << 20, 500, seed=0, step=1, t=0)
  for kwargs in ({"seed": 1, "step": 1, "t": 0}, {"seed": 0, "step": 2, "t": 0}, {"seed": 0, "step": 1, "t": 1}):
    other = _ops.dnc_sample(1 << 20, 500, **kwargs)
    assert not np.array_equal(base, other)
  # a prefix of a longer sample: P(0), ..., P(b' - 1)
  assert np.array_equal(_ops.dnc_sample(1 << 20, 1000, seed=0, step=1, t=0)[:500], base)


def test_sampler_matches_a_scalar_transcription():
  mask64 = (1 << 64) - 1

  def sm(z):
    z = (z + 0x9E3779B97F4A7C15) & mask64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & mask64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & mask64
    return z ^ (z >> 31)

  for domain, seed, step, t in ((1000, 5, 9, 2), (2 ** 33 + 7, 2 ** 64 - 1, 123456, 0), (2, 0, 0, 0)):
    key = sm(sm(sm(seed) ^ step) ^ t)
    w = max(2, (domain - 1).bit_length())
    h = (w + (w & 1)) // 2
    expected = []
    for x in range(min(50, domain)):
      y = x
      while True:
        L, R = y >> h, y & ((1 << h) - 1)
        for r in range(4):
          L, R = R, L ^ (sm(key ^ (r << 48) ^ R) & ((1 << h) - 1))
        y = (L << h) | R
        if y < domain:
          break
      expected.append(y)
    assert _ops.dnc_sample(domain, 50, seed, step, t).tolist() == expected


# ---------------------------------------------------------------------------- #
# Scores and Jacobi

@pytest.mark.parametrize("m", [2, 3, 7, 8, 17, 32])
def test_scores_match_the_svd_of_the_centred_sample(m):
  rng = np.random.default_rng(m)
  X = rng.standard_normal((m, 300)).astype(np.float32).astype(np.float64)
  X[0] += 4.0   # a clear top direction
  D = ((X[:, None, :] - X[None, :, :]) ** 2).sum(axis=2)
  scores = _ops.dnc_scores(D)
  centred = X - X.mean(axis=0)
  U, S, _ = np.linalg.svd(centred, full_matrices=False)
  assert np.allclose(scores, U[:, 0] ** 2, rtol=1e-9, atol=1e-12)
  # the paper's score <x_i - mu, v>^2 = lambda_1 u_i^2 ranks the rows the same way
  paper = (centred @ np.linalg.svd(centred)[2][0]) ** 2
  assert np.allclose(paper, S[0] ** 2 * scores, rtol=1e-8, atol=1e-9)


@pytest.mark.parametrize("m", list(range(2, 41)))
def test_jacobi_matches_lapack_on_random_psd_matrices(m):
  rng = np.random.default_rng(100 + m)
  A = rng.standard_normal((m, m + 3))
  B = A @ A.T
  lam, V = _ops.dnc_eigh(B)
  ref = np.linalg.eigvalsh(B)
  assert np.allclose(np.sort(lam), ref, rtol=1e-10, atol=1e-10 * ref.max())
  assert np.allclose(V.T @ V, np.eye(m), atol=1e-10)
  k = int(np.argmax(lam))
  w, U = np.linalg.eigh(B)
  assert abs(abs(float(V[:, k] @ U[:, -1])) - 1.0) < 1e-10


def test_scores_of_one_or_no_row_are_zero():
  assert _ops.dnc_scores(np.zeros((1, 1))).tolist() == [0.0]
  assert _ops.dnc_scores(np.zeros((0, 0))).tolist() == []
  assert _ops.dnc_scores(np.zeros((3, 3))).tolist() == [1.0, 0.0, 0.0]   # no spread: B = 0, V = I, the tie goes to column 0


# ---------------------------------------------------------------------------- #
# Hand cases

def _rows(n, d, seed):
  return torch.randn(n, d, generator=torch.Generator().manual_seed(seed))


def test_f_zero_is_the_average():
  G = _rows(6, 1003, 1)
  out = _ops.torch_dnc(G, 0, 2, 100, 1.0, 0, 1)
  assert torch.equal(out, _ops.selection_mean(G, np.ones(6, dtype=bool)))
  assert torch.allclose(out, G.mean(dim=0), atol=1e-6)
  assert torch.equal(_ops.host_dnc(G, 0, 2, 100, 1.0, 0, 1), out)


def test_one_outlier_along_a_direction_is_removed():
  G = _rows(9, 5000, 2) * 0.1
  G[4] += 3.0
  out, dists, (masks, good) = _ops.torch_dnc(G, 2, 1, 1000, 0.5, 0, 1, return_details=True)
  assert dists.shape == (1, 9, 9)
  assert good.tolist() == [i != 4 for i in range(9)]
  assert torch.equal(out, _ops.selection_mean(G, good))


def test_non_finite_rows_are_dropped_first():
  G = _rows(8, 2000, 3)
  G[2, ::3] = float("nan")
  G[6, 1::3] = float("inf")
  G[6, 2::3] = float("-inf")
  out, dists, (masks, good) = _ops.torch_dnc(G, 2, 1, 2000, 1.0, 0, 1, return_details=True)
  assert not good[2] and not good[6] and good.sum() == 6
  assert bool(torch.isfinite(out).all())
  # only one NaN coordinate: row 2 has 7 non-finite distances, the others one (to row 2); row 2 goes, then all is finite
  H = _rows(5, 100, 4)
  H[1, 10] = float("nan")
  _, _, (_, good) = _ops.torch_dnc(H, 1, 1, 100, 1.0, 0, 1, return_details=True)
  assert not good[1] and good.sum() == 4


def test_non_finite_ties_drop_the_highest_index():
  D = np.zeros((1, 4, 4))
  D[0, 0, 1] = D[0, 1, 0] = np.inf   # rows 0 and 1 both have one non-finite distance: row 1 goes, then everything is finite
  masks, good = _ops.dnc_select(D, 1)
  assert masks[0].tolist() == [True, False, True, True]


def test_the_good_set_is_the_intersection_over_iterations():
  rng = np.random.default_rng(5)
  X = rng.standard_normal((7, 40))
  dists = []
  for out in (1, 3, 5):
    Y = X.copy()
    Y[out] += 10 * rng.standard_normal(40)
    dists.append(((Y[:, None, :] - Y[None, :, :]) ** 2).sum(axis=2))
  masks, good = _ops.dnc_select(np.stack(dists), 1)
  assert [int(np.flatnonzero(~m)[0]) for m in masks] == [1, 3, 5]
  assert good.tolist() == [True, False, True, False, True, False, True]
  G = torch.randn(7, 3000, generator=torch.Generator().manual_seed(6))
  G[[1, 5]] += 5.0 * torch.randn(2, 3000, generator=torch.Generator().manual_seed(7))
  _, _, (masks, good) = _ops.torch_dnc(G, 2, 3, 400, 1.0, 0, 1, return_details=True)
  assert masks.shape == (3, 7) and np.array_equal(good, masks.all(axis=0)) and not good[1] and not good[5]


def test_removes_every_min_max_row():
  n, f, d = 10, 3, 20000
  G = torch.randn(n, d, generator=torch.Generator().manual_seed(8)) * 0.5 + 1.0
  _ops.torch_craft_byzantine_(G, list(range(n - f, n)), "min-max", deviation="std")
  _, _, (_, good) = _ops.torch_dnc(G, f, 1, 10000, 1.0, 0, 1, return_details=True)
  assert good.tolist() == [True] * (n - f) + [False] * f


# ---------------------------------------------------------------------------- #
# Host library

@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("n,d,b,T", [(3, 101, 50, 1), (8, 4003, 1000, 3), (17, 999, 5000, 2)])
def test_host_library_matches_the_torch_reference(n, d, b, T, dtype):
  G = _rows(n, d, n + d).to(dtype)
  G[n - 1] = G[n - 1] * 20 + 3
  out, dists, (masks, good) = _ops.host_dnc(G, 1, T, b, 1.0, 11, 5, return_details=True)
  ref, ref_dists, (ref_masks, ref_good) = _ops.torch_dnc(G, 1, T, b, 1.0, 11, 5, return_details=True)
  assert dists.dtype == dtype and dists.shape == (T, n, n)
  assert torch.allclose(dists, ref_dists, rtol=1e-5 if dtype == torch.float32 else 1e-12)
  assert np.array_equal(masks, ref_masks) and np.array_equal(good, ref_good)
  assert torch.equal(out, ref)   # the same mask: the same bits


def test_gar_object_counts_its_calls():
  gar = aggregators.instantiate("dnc", 6, 1, ["iterations:2", "subsample:64", "seed:9"])
  G = _rows(6, 500, 12)
  first, second = gar.aggregate(G), gar.aggregate(list(G))
  assert torch.equal(first, _ops.host_dnc(G, 1, 2, 64, 1.0, 9, 1))
  assert torch.equal(second, _ops.host_dnc(G, 1, 2, 64, 1.0, 9, 2))
  assert torch.equal(gar.aggregate(G, step=1), first)
  assert repr(gar.fused_spec()) == "FusedSpec(rule='dnc', n=6, f=1, m=0, beta=0, iterations=2, subsample=64, c=1.0, seed=9)"
  assert FusedSpec.RULES.index("dnc") == 10 and "dnc" in FusedSpec.RULES_WITH_F
  assert gar.fused_spec().with_mix("nnm").subsample == 64 and gar.fused_spec().removed == 1


def test_argument_errors():
  for args in (["iterations:0"], ["iterations:9"], ["subsample:0"], ["subsample:1048577"], ["c:-1"], ["c:inf"], ["seed:-1"],
               ["seed:18446744073709551616"], ["iterations:4", "c:1.0"]):
    with pytest.raises(tools.UserException):
      aggregators.instantiate("dnc", 7, 2, args)
  for n, f in ((4, 2), (3, -1)):
    with pytest.raises(tools.UserException):
      aggregators.instantiate("dnc", n, f, [])
  assert _ops.check_dnc(7, 3, 2, 10, 0.5, 0)[4] == 1 and _ops.check_dnc(7, 2, 3, 10, 1.0, 0)[4] == 2
  assert _ops.check_dnc(10, 3, 1, 10, 1 / 3 * 3, 0)[4] == math.floor(1 / 3 * 3 * 3)
  with pytest.raises(tools.UserException):
    _ops.torch_dnc(torch.zeros(5, 10), 1, 1, 10, 1.0, 0, 1, domain=11)
  with pytest.raises(tools.UserException):
    _ops.dnc_sample(0, 10, 0, 0, 0)
  for step in (-1, 1 << 63, 1.5):   # the kernels take a signed 64-bit step key >= 0: every back-end has the same domain
    with pytest.raises(tools.UserException):
      _ops.dnc_sample(100, 10, 0, step, 0)
    with pytest.raises(tools.UserException):
      _ops.torch_dnc(torch.zeros(5, 10), 1, 1, 10, 1.0, 0, step)
    with pytest.raises(tools.UserException):
      _ops.host_dnc(torch.zeros(5, 10), 1, 1, 10, 1.0, 0, step)


# ---------------------------------------------------------------------------- #
# Engines, checkpoints, runner

def test_host_engine_end_to_end_and_resume():
  layout = FlatLayout()
  layout.add("w", (70, 3))
  layout.freeze()
  gar = aggregators.instantiate("dnc", 5, 1, ["iterations:2", "subsample:50"])
  gen = torch.Generator().manual_seed(13)
  grads = [torch.randn(5, layout.padded_size, generator=gen) for _ in range(4)]

  def engine():
    return HostAggregation(gar, layout, 5, build(optimizers, "optimizer", "sgd", []), device="cpu")
  straight = engine()
  for k, G in enumerate(grads):
    straight.grads.copy_(G)
    straight.step(0.1)
    assert torch.equal(straight.last_aggregate, _ops.host_dnc(G, 1, 2, 50, 1.0, 0, k + 1))
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
  assert torch.equal(resumed.params, straight.params)


def _run(args, timeout=300):
  env = dict(os.environ, AGB_NUM_THREADS="2", OMP_NUM_THREADS="2")
  proc = subprocess.run([sys.executable, str(ROOT / "runner.py")] + args, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=timeout, env=env, cwd=str(ROOT))
  return proc.returncode, proc.stdout.decode(errors="replace")


def test_runner_trains_and_resumes_from_a_checkpoint(tmp_path):
  def args(directory, steps):
    return LOCAL + ["--experiment", "mnist", "--aggregator", "dnc", "--aggregator-args", "iterations:2", "subsample:500", "--nb-workers", "5",
                    "--nb-decl-byz-workers", "1", "--max-step", str(steps), "--seed", "3", "--learning-rate-args", "initial-rate:0.05",
                    "--evaluation-file", "-", "--summary-dir", "-", "--evaluation-delta", "1000", "--evaluation-period", "-1",
                    "--checkpoint-dir", str(directory), "--checkpoint-period", "-1", "--checkpoint-delta", "2"]
  losses = lambda out: dict(re.findall(r"Step (\d+): total loss = ([0-9.eE+-]+|NaN)", out))
  code, straight = _run(args(tmp_path / "straight", 4))
  assert code == 0, straight
  code, out = _run(args(tmp_path / "resumed", 2))
  assert code == 0, out
  code, resumed = _run(args(tmp_path / "resumed", 2))   # --max-step counts the steps of this run
  assert code == 0, resumed
  # the runner does not restore the order of the training data, so the losses after the resume are not compared; the engine test
  # above checks that resumed updates draw the same samples
  got = losses(resumed)
  assert "3" in got and "0" not in got and all(math.isfinite(float(x)) for x in got.values()), resumed   # resumed from step 2
  assert len(losses(straight)) == 4

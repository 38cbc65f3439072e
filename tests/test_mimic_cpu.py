"""The mimic attack (Karimireddy, He & Jaggi, ICLR 2022) on the CPU: the torch reference against an independent float64 transcription of
the online power iteration, the argument checks, the host engine end to end (with its checkpoint) and the runner CLI."""

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

ROOT = pathlib.Path(__file__).resolve().parent.parent
LOCAL = ["--server", '{"local": ["127.0.0.1:7000"]}', "--ps-job-name", "local", "--wk-job-name", "local", "--ev-job-name", "local", "--no-wait"]


def oracle_trajectory(rows_per_step, byz, warmup):
  """float64 transcription of the recursion: per step, the honest rows h (ascending slots), mu, s_i = <h_i - mu, z>, u = mean_i s_i (h_i - mu),
  y = (t z + u) / (t + 1), z = y / ||y||, i* = argmax_i <h_i, y> (finite, lower slot on ties). -> (i* per step, z after the warm-up)."""
  d = rows_per_step[0].shape[1]
  z = np.full(d, 1.0 / math.sqrt(d))
  t, target, targets = 0, None, []
  for G in rows_per_step:
    honest_ids = [i for i in range(G.shape[0]) if i not in byz]
    if t < warmup:
      X = G[honest_ids].astype(np.float64)
      dev = X - X.mean(axis=0)
      s = dev @ z
      y = (t * z + (s[:, None] * dev).mean(axis=0)) / (t + 1)
      norm = np.linalg.norm(y)
      if norm > 0 and np.isfinite(norm):
        z = y / norm
        q = X @ y
        target = honest_ids[int(np.argmax(np.where(np.isfinite(q), q, -np.inf)))]
      t += 1
    targets.append(honest_ids[0] if target is None else target)
  return targets, z


def _rows(rng, n, d, spread, base=None):
  """n rows whose honest spread lies mostly along one direction `base` (a clear top principal component), plus small noise."""
  base = rng.standard_normal(d) if base is None else base
  coef = np.linspace(-spread, spread, n)
  rng.shuffle(coef)
  return (coef[:, None] * base[None, :] + 0.05 * rng.standard_normal((n, d))).astype(np.float32), base


@pytest.mark.parametrize("n,k,d", [(3, 1, 37), (8, 2, 1001), (9, 1, 515), (17, 2, 203)])
def test_reference_follows_the_float64_oracle(n, k, d):
  rng = np.random.default_rng(n * 1000 + d)
  byz = list(range(n - k, n))
  warmup = 12
  base = rng.standard_normal(d)
  steps = [_rows(rng, n, d, 1.0 + 0.1 * i, base)[0] for i in range(20)]
  expected, z64 = oracle_trajectory(steps, byz, warmup)
  state = _ops.mimic_state(d)
  got = []
  for i, X in enumerate(steps):
    G = torch.from_numpy(X.copy())
    details = _ops.torch_mimic_step_(G, byz, state, warmup, return_details=True)
    assert (details is None) == (i >= warmup)
    target = int(state["istar"][0])
    got.append(target)
    for b in byz:
      assert torch.equal(G[b], G[target])   # bit for bit
    honest = [j for j in range(n) if j not in byz]
    assert torch.equal(G[honest], torch.from_numpy(X[honest]))
  assert got == expected
  assert state["t"] == warmup
  z = state["z"].double().numpy()
  assert np.linalg.norm(z - z64) <= 1e-5 * np.linalg.norm(z64)


def test_state_is_frozen_after_the_warmup():
  rng = np.random.default_rng(5)
  X, _ = _rows(rng, 6, 64, 2.0)
  state = _ops.mimic_state(64)
  for _ in range(3):
    _ops.torch_mimic_step_(torch.from_numpy(X.copy()), [5], state, 3)
  z, target = state["z"].clone(), int(state["istar"][0])
  Y, _ = _rows(rng, 6, 64, 5.0)
  G = torch.from_numpy(Y.copy())
  assert _ops.torch_mimic_step_(G, [5], state, 3, return_details=True) is None
  assert state["t"] == 3 and torch.equal(state["z"], z) and int(state["istar"][0]) == target
  assert torch.equal(G[5], G[target])


def test_degenerate_norm_keeps_the_state():
  G = torch.ones((4, 16))   # identical honest rows: u = 0, y = 0 at t = 0
  state = _ops.mimic_state(16)
  z = state["z"].clone()
  s, q, norm2, inv = _ops.torch_mimic_step_(G, [3], state, 5, return_details=True)
  assert norm2 == 0 and inv == 0 and s == [0.0, 0.0, 0.0]
  assert state["t"] == 1 and torch.equal(state["z"], z) and int(state["istar"][0]) == -1
  assert torch.equal(G[3], G[0])   # no target yet: the first honest slot


def test_target_and_padding():
  # the spread lies along the first two real coordinates, where row 0 reaches furthest; padding coordinates stay 0
  mask = torch.tensor([True, True, False, True, False, False, True, True])
  state = _ops.mimic_state(8, mask=mask)
  assert torch.equal(state["z"][~mask], torch.zeros(3)) and float(state["z"][0]) == float(np.float32(1 / math.sqrt(5)))
  G = torch.zeros((4, 8))
  G[:3, mask] = torch.tensor([[3., 1., 0., 0., 0.], [-3., -1., 0., 0., 0.], [0., 0., 1., 0., 0.]])
  _ops.torch_mimic_step_(G, [3], state, 10)
  assert torch.equal(state["z"][~mask], torch.zeros(3))
  assert int(state["istar"][0]) == 0 and torch.equal(G[3], G[0])


def test_argument_checks():
  with pytest.raises(tools.UserException):
    attacks.instantiate("mimic", 4, 3, [])           # one honest row
  with pytest.raises(tools.UserException):
    attacks.instantiate("mimic", 6, 1, ["warmup:0"])
  with pytest.raises(tools.UserException):
    attacks.instantiate("mimic", 6, 1, ["warmup:1.5"])
  with pytest.raises(tools.UserException):
    attacks.instantiate("mimic", 6, 1, ["deviation:std"])
  attack = attacks.instantiate("mimic", 6, 1, [])
  assert attack.mode == "mimic" and attack.warmup == 100 and attack.coef is None and attack.omniscient
  assert attacks.instantiate("mimic", 6, 2, ["warmup:7"]).warmup == 7
  with pytest.raises(tools.UserException):
    _ops.check_mimic(5, [1, 2, 3, 4], 3)
  with pytest.raises(tools.UserException):
    _ops.check_mimic(5, [4], 0)
  with pytest.raises(tools.UserException):
    _ops.check_mimic(5, [4], True)
  with pytest.raises(tools.UserException):
    _ops.torch_mimic_step_(torch.zeros((5, 4), dtype=torch.float64), [4], _ops.mimic_state(4), 3)


def _manager(n, k, warmup, seed=1, experiment_args=("batch-size:16", "dirichlet:0.5")):
  experiment = experiments.instantiate("mnist", list(experiment_args))
  attack = attacks.instantiate("mimic", n, k, ["warmup:%d" % warmup])
  return Manager(experiment, aggregators.instantiate("median", n, k, []), n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu", attack=attack,
                 nb_real_byz=k, seed=seed)


def test_host_engine_trains_and_checkpoints_the_state():
  n, k = 6, 2
  mgr = _manager(n, k, warmup=2)
  assert mgr.aggregation.name == "host" and mgr.byzantine_slots == [4, 5]
  for step in range(3):
    loss = float(mgr.train())
    assert math.isfinite(loss)
    rows = mgr.aggregation.visible_rows()
    target = int(mgr.aggregation.attack_state["istar"][0])
    assert target in range(4) and torch.equal(rows[4], rows[target]) and torch.equal(rows[5], rows[target])
    assert (mgr.aggregation.last_craft is None) == (step >= 2)
  saved = mgr.state_dict()
  assert saved["aggregation"]["attack_state"]["t"] == 2 and saved["aggregation"]["attack_state"]["istar"] == target
  other = _manager(n, k, warmup=2)
  other.load_state_dict(saved)
  state = other.aggregation.attack_state
  assert state["t"] == 2 and int(state["istar"][0]) == target and torch.equal(state["z"], mgr.aggregation.attack_state["z"])
  del saved["aggregation"]["attack_state"]
  other.load_state_dict(saved)   # an older checkpoint: the warm-up starts again
  assert other.aggregation.attack_state["t"] == 0


# ---------------------------------------------------------------------------- #
# Runner CLI

def _run(args, timeout=300):
  env = dict(os.environ, AGB_NUM_THREADS="2", OMP_NUM_THREADS="2")
  proc = subprocess.run([sys.executable, str(ROOT / "runner.py")] + args, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=timeout, env=env, cwd=str(ROOT))
  return proc.returncode, proc.stdout.decode(errors="replace")


def test_runner_dirichlet_mimic_bucketing_krum(tmp_path):
  evaluation = tmp_path / "eval"
  args = LOCAL + ["--experiment", "mnist", "--experiment-args", "batch-size:16", "dirichlet:0.3", "--aggregator", "krum", "--nb-workers", "10",
                  "--nb-decl-byz-workers", "1", "--nb-real-byz-workers", "2", "--pre-aggregation", "bucketing", "--bucket-size", "2",
                  "--attack", "mimic", "--attack-args", "warmup:2", "--max-step", "4", "--seed", "3", "--learning-rate-args", "initial-rate:0.05",
                  "--evaluation-file", str(evaluation), "--summary-dir", "-", "--evaluation-delta", "2", "--evaluation-period", "-1",
                  "--checkpoint-period", "-1", "--checkpoint-delta", "1000"]
  code, out = _run(args)
  assert code == 0, out
  losses = re.findall(r"Step \d+: total loss = ([0-9.eE+-]+|NaN)", out)
  assert len(losses) == 4 and all(math.isfinite(float(x)) for x in losses), out
  assert len(re.findall(r"Worker \d+: \d+ training samples of \d+ classes", out)) == 10, out
  assert evaluation.is_file() and evaluation.read_text().strip(), out
  code, out = _run(args[:args.index("warmup:2")] + ["warmup:-1"] + args[args.index("warmup:2") + 1:])
  assert code != 0 and "warmup" in out

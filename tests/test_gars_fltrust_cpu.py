"""FLTrust (`aggregators/fltrust.py`) on the CPU: the torch and host back-ends against a float64 oracle of the paper's formula, the
shared coefficient arithmetic, its properties, the argument checks, the root dataset and end-to-end runs."""

import os
import pathlib
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from aggregathor_b200 import aggregators, attacks, experiments, tools
from aggregathor_b200.aggregators import FusedSpec, _ops
from aggregathor_b200.engine.trainer import Manager

ROOT = pathlib.Path(__file__).resolve().parent.parent


def _oracle(G, r):
  """The paper's formula in float64: sum ReLU(cos(x_i, r)) (||r|| / ||x_i||) x_i / sum ReLU(cos), +0 when no row is trusted."""
  G, r = np.asarray(G, dtype=np.float64), np.asarray(r, dtype=np.float64)
  nr = np.linalg.norm(r)
  out, total = np.zeros(G.shape[1]), 0.0
  for x in G:
    nx = np.linalg.norm(x)
    if not (np.isfinite(nx) and nx > 0 and np.isfinite(nr) and nr > 0):
      continue
    ts = max(0.0, float(x @ r) / (nx * nr))
    out += ts * (nr / nx) * x
    total += ts
  return out / total if total > 0 else out


def _rows(n, d, seed, dtype=torch.float32):
  gen = torch.Generator().manual_seed(seed)
  r = torch.randn(d, generator=gen, dtype=torch.float64)
  G = 0.5 * r + torch.randn((n, d), generator=gen, dtype=torch.float64) * torch.rand((n, 1), generator=gen, dtype=torch.float64) * 2
  return G.to(dtype), r.to(dtype)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("n", [1, 2, 5, 8, 19, 32])
def test_backends_match_float64_oracle(n, dtype):
  G, r = _rows(n, 1003, n, dtype)
  G[n // 2] = -3 * G[n // 2]   # at least one row pointing away from r when n > 1
  want = _oracle(G.numpy(), r.numpy())
  tol = 1e-5 if dtype == torch.float32 else 1e-12
  scale = float(torch.linalg.norm(r.double()))
  for out in (_ops.torch_fltrust(G, r), _ops.host_fltrust(G, r), aggregators.instantiate("fltrust", n, 0, []).aggregate(G, root=r)):
    assert out.dtype == dtype
    assert np.abs(out.double().numpy() - want).max() <= tol * scale


@pytest.mark.parametrize("n", [1, 3, 8, 32])
def test_same_sums_give_the_same_bits(n):
  G, r = _rows(n, 517, 7 + n)
  G[0, 3] = float("nan")
  sums = _ops.host_fltrust_sums(G, r)
  torch_out, *tdetails = _ops.torch_fltrust(G, r, sums=sums, return_details=True)
  host_out, *hdetails = _ops.host_fltrust(G, r, return_details=True)
  assert torch.equal(torch_out, host_out)
  assert np.array_equal(tdetails[3], hdetails[3]) and tdetails[3].dtype == np.float32
  # the coefficients against a literal transcription of the stated order of operations
  P, N, N0 = (np.asarray(v, dtype=np.float64) for v in sums)
  s0 = np.sqrt(float(N0))
  ts = []
  for i in range(n):
    with np.errstate(all="ignore"):
      t = P[i] / (np.sqrt(N[i]) * s0)
    ts.append(t if np.isfinite(t) and t > 0 else 0.0)
  S = 0.0
  for v in ts:
    S += v
  a = [np.float32(((v * s0) / np.sqrt(N[i])) / S) if S != 0 and v > 0 else np.float32(0) for i, v in enumerate(ts)]
  assert np.array_equal(np.array(a, dtype=np.float32), hdetails[3])
  # y from +0 in worker order, one rounding per product and sum, the zero-weight rows skipped
  y = np.zeros(G.shape[1], dtype=np.float32)
  for i in range(n):
    if a[i] != 0:
      y = (y + (np.float32(a[i]) * G[i].numpy()).astype(np.float32)).astype(np.float32)
  assert np.array_equal(y, host_out.numpy())


def test_negative_cosine_gets_no_weight():
  G, r = _rows(5, 64, 1)
  G[2] = -G[2].abs() * r.sign()
  _, P, N, N0, a = _ops.host_fltrust(G, r, return_details=True)
  assert P[2] < 0 and a[2] == 0 and (a[[0, 1, 3, 4]] > 0).all()
  assert torch.equal(_ops.host_fltrust(G, r), _ops.host_fltrust(G[[0, 1, 3, 4]], r))


def test_scaling_a_row_leaves_the_output_unchanged():
  G, r = _rows(6, 300, 2)
  scaled = G.clone()
  scaled[1] *= 1000.0
  scaled[4] *= 1e-3
  a, b = _ops.host_fltrust(G, r), _ops.host_fltrust(scaled, r)
  assert torch.allclose(a, b, rtol=1e-5, atol=1e-6 * float(torch.linalg.norm(r)))


def test_no_trusted_row_gives_positive_zero():
  G, r = _rows(4, 100, 3)
  for rows, root in ((-G.abs() * r.sign(), r), (G, torch.zeros_like(r)), (G, torch.full_like(r, float("nan")))):
    for out in (_ops.host_fltrust(rows, root), _ops.torch_fltrust(rows, root)):
      assert torch.equal(out, torch.zeros_like(out)) and not torch.signbit(out).any()


def test_non_finite_rows_are_skipped():
  G, r = _rows(6, 200, 4)
  bad = G.clone()
  bad[1, 7] = float("nan")
  bad[3, 0] = float("inf")
  bad[5, :] = -float("inf")
  for backend in (_ops.host_fltrust, _ops.torch_fltrust):
    out, want = backend(bad, r), backend(G[[0, 2, 4]], r)
    assert torch.isfinite(out).all() and torch.allclose(out, want, rtol=1e-6, atol=1e-7)
  # given the same sums of the finite rows, the same bits
  P, N, N0 = _ops.host_fltrust_sums(bad, r)
  keep = [0, 2, 4]
  assert torch.equal(_ops.torch_fltrust(bad, r, sums=(P, N, N0)), _ops.torch_fltrust(G[keep], r, sums=(P[keep], N[keep], N0)))


@pytest.mark.parametrize("seed", range(5))
def test_output_norm_is_bounded_by_the_root_norm(seed):
  G, r = _rows(9, 777, 10 + seed)
  G[::2] *= 50.0
  for out in (_ops.host_fltrust(G, r), _ops.torch_fltrust(G, r)):
    assert float(torch.linalg.norm(out.double())) <= float(torch.linalg.norm(r.double())) * (1 + 1e-6)


def test_rule_ids_and_spec():
  assert FusedSpec.RULES.index("fltrust") == 12
  assert FusedSpec.RULES[:12] == ("average", "average-nan", "median", "averaged-median", "krum", "bulyan", "trimmed-mean", "mda",
                                  "geometric-median", "centered-clipping", "dnc", "smea")
  assert "fltrust" not in FusedSpec.RULES_WITH_F
  gar = aggregators.instantiate("fltrust", 8, 2, ["root-size:50"])
  spec = gar.fused_spec()
  assert (spec.rule, spec.n, spec.rule_id, gar.needs_root, gar.root_size) == ("fltrust", 8, 12, True, 50)
  assert aggregators.instantiate("fltrust", 8, 7, []).root_size == 100


def test_argument_errors():
  for args in (["root-size:0"], ["root-size:-3"], ["root-size:x"], ["root-size:2.5"]):
    with pytest.raises(tools.UserException):
      aggregators.instantiate("fltrust", 8, 2, args)
  with pytest.raises(tools.UserException):
    aggregators.instantiate("fltrust", 4, 4, [])
  gar = aggregators.instantiate("fltrust", 4, 1, [])
  with pytest.raises(tools.UserException, match="root"):
    gar.aggregate(torch.ones(4, 8))


@pytest.mark.parametrize("mix", ["nnm", "arc", "arc+nnm", "bucketing"])
def test_pre_aggregation_is_refused(mix):
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate("fltrust", 4 if mix == "bucketing" else 8, 2 if mix != "bucketing" else 1, [])
  with pytest.raises(tools.UserException, match="pre-aggregation"):
    Manager(experiment, gar, 8, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu", pre_aggregation=mix,
            bucket_size=2 if mix == "bucketing" else None)


def test_worker_momentum_and_small_root_are_refused():
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  with pytest.raises(tools.UserException, match="worker-momentum"):
    Manager(experiment, aggregators.instantiate("fltrust", 4, 1, []), 4, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu", worker_momentum=0.9)
  with pytest.raises(tools.UserException, match="batch-size"):
    Manager(experiment, aggregators.instantiate("fltrust", 4, 1, ["root-size:8"]), 4, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu")


def test_root_subset():
  plain = experiments.instantiate("mnist", ["batch-size:16", "seed:3"])
  skewed = experiments.instantiate("mnist", ["batch-size:16", "seed:3", "dirichlet:0.1"])
  other = experiments.instantiate("mnist", ["batch-size:16", "seed:4"])
  idx = plain.root_indices(100)
  assert len(idx) == 100 and len(np.unique(idx)) == 100 and (np.diff(idx) > 0).all()
  assert np.array_equal(idx, plain.root_indices(100)) and np.array_equal(idx, skewed.root_indices(100))
  assert not np.array_equal(idx, other.root_indices(100))
  skewed.train_stream(0, 4, "cpu")   # the Dirichlet partition draws nothing from the root's generator
  assert np.array_equal(idx, skewed.root_indices(100))
  # the stream serves root samples only
  keys = {plain.data.x_train[i].tobytes() for i in idx}
  stream = plain.root_stream(100, "cpu")
  try:
    for _ in range(10):
      x, y = next(stream)
      assert x.shape[0] == 16 and all(row.numpy().tobytes() in keys for row in x)
  finally:
    stream.close()


def test_root_stream_is_never_poisoned():
  experiment = experiments.instantiate("mnistAttack", ["batch-size:16"])
  clean = {experiment.data.x_train[i].tobytes() + experiment.data.y_train[i].tobytes() for i in experiment.root_indices(64)}
  stream = experiment.root_stream(64, "cpu")
  try:
    for _ in range(6):
      x, y = next(stream)
      assert all(row.numpy().tobytes() + label.numpy().tobytes() in clean for row, label in zip(x, y))
  finally:
    stream.close()


def _manager(gar_name, n, f, attack=None, real=0, gar_args=()):
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate(gar_name, n, f, list(gar_args))
  return Manager(experiment, gar, n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu", attack=attack, nb_real_byz=real)


def test_fltrust_survives_flip_average_does_not():
  robust = _manager("fltrust", 8, 2, attacks.instantiate("flip", 8, 2, ["factor:-10"]), 2, ["root-size:100"])
  assert robust.aggregation.name == "host" and robust.root_ctx is not None
  first = float(robust.train())
  for _ in range(25):
    last = float(robust.train())
  assert last == last and last < first
  assert robust.evaluate()["top1-X-acc"] > 0.5
  assert float(torch.linalg.norm(robust.aggregation.last_aggregate)) <= float(torch.linalg.norm(robust.aggregation.root)) * (1 + 1e-6)
  naive = _manager("average", 8, 2, attacks.instantiate("flip", 8, 2, ["factor:-10"]), 2)
  for _ in range(25):
    loss = float(naive.train())
  assert not (loss == loss and naive.evaluate()["top1-X-acc"] > 0.5 and loss < first)


def _run(args, timeout=600, launcher=None):
  env = dict(os.environ, AGB_NUM_THREADS="2", OMP_NUM_THREADS="2")
  cmd = (launcher or [sys.executable]) + [str(ROOT / "runner.py")] + args
  proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=timeout, env=env, cwd=str(ROOT))
  return proc.returncode, proc.stdout.decode(errors="replace")


COMMON = ["--experiment", "mnist", "--aggregator", "fltrust", "--max-step", "8", "--learning-rate-args", "initial-rate:0.05",
          "--evaluation-delta", "1000", "--evaluation-period", "-1", "--summary-dir", "-"]


def test_runner_fltrust_under_flip():
  local = ["--server", '{"local": ["127.0.0.1:7000"]}', "--ps-job-name", "local", "--wk-job-name", "local", "--ev-job-name", "local", "--no-wait"]
  code, out = _run(local + COMMON + ["--nb-workers", "8", "--nb-decl-byz-workers", "2", "--nb-real-byz-workers", "2", "--attack", "flip",
                                     "--attack-args", "factor:-10"])
  assert code == 0, out
  losses = [float(x) for x in re.findall(r"Step \d+: total loss = ([0-9.eE+-]+)", out)]
  assert len(losses) == 8 and losses[-1] < losses[0]
  code, out = _run(local + COMMON + ["--nb-workers", "4", "--pre-aggregation", "nnm", "--nb-decl-byz-workers", "1"])
  assert code != 0 and "pre-aggregation" in out and "Traceback" not in out


def test_two_process_gloo_root_from_rank_0():
  port = 29500 + (os.getpid() + 7) % 400
  launcher = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", str(port)]
  args = ["--server", '{"ps": ["127.0.0.1:7000"], "workers": ["127.0.0.1:7001", "127.0.0.1:7002"], "eval": ["127.0.0.1:7000"]}', "--no-wait",
          "--nb-workers", "4", "--debug-checksum"] + COMMON
  code, out = _run(args, launcher=launcher)
  assert code == 0, out
  assert "Step 7: total loss" in out and "Replica divergence" not in out

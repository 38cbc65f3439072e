"""Worker momentum on the CPU: the torch reference against a step-by-step fp32 NumPy evaluation, the option checks, the switched-off
default, a Byzantine worker's momentum under `flip`, and checkpoint / resume of the momenta on the host engine."""

import numpy as np
import pytest
import torch

from aggregathor_b200 import aggregators, attacks, experiments, tools
from aggregathor_b200.aggregators import _ops
from aggregathor_b200.cli import runner
from aggregathor_b200.engine.trainer import Manager


def _equal_bits(a, b):
  a, b = torch.as_tensor(a).cpu(), torch.as_tensor(b).cpu()
  assert a.dtype == b.dtype and a.shape == b.shape
  nan = torch.isnan(a)
  assert torch.equal(nan, torch.isnan(b))
  assert torch.equal(a[~nan].view(torch.int32), b[~nan].view(torch.int32))


def _rows(w, d, seed):
  gen = torch.Generator().manual_seed(seed)
  G = torch.randn(w, d, generator=gen) * 3
  G[0, 5::37] = float("nan")
  G[-1, 7::31] = float("inf")
  G[-1, 11::29] = float("-inf")
  G[0, 13::23] = 3e38
  return G


@pytest.mark.parametrize("coefs", [(0.9, 0.0), (0.9, 0.1), (0.5, 0.5), (0.0, 0.3), (0.99, 0.999), (0.1, 0.0)])
def test_reference_matches_fp32_numpy(coefs):
  beta, c = _ops.check_worker_momentum(*coefs)
  assert beta == float(np.float32(coefs[0])) and c == float(np.float32(1.0 - float(np.float32(coefs[1]))))
  w, d = 4, 1001
  M = torch.zeros(w, d)
  m = np.zeros((w, d), dtype=np.float32)
  for step in range(4):
    G = _rows(w, d, seed=step)
    g = G.numpy().copy()
    _ops.torch_worker_momentum_(G, M, beta, c)
    with np.errstate(over="ignore", invalid="ignore"):
      m = np.float32(beta) * m + np.float32(c) * g   # each NumPy fp32 operation is rounded once
    _equal_bits(M, torch.from_numpy(m))
    _equal_bits(G, torch.from_numpy(m))
  assert bool(torch.isnan(M).any())


def test_double_rows_use_the_coefficients_as_rounded():
  beta, c = _ops.check_worker_momentum(0.9, 0.1)
  G, M = torch.randn(2, 50, dtype=torch.float64), torch.randn(2, 50, dtype=torch.float64)
  expect = M * beta + G * c
  from aggregathor_b200.ops import gar as gar_ops
  gar_ops.worker_momentum_(G, M, beta, c)
  assert torch.equal(M, expect) and torch.equal(G, expect)


def test_option_errors():
  for beta, dampening in ((1.0, 0.0), (-0.1, 0.0), (0.5, 1.0), (0.5, -1e-3), (float("nan"), 0.0), (float("inf"), 0.0), (0.5, float("nan")),
                          (0.99999999, 0.0), ("x", 0.0)):
    with pytest.raises(tools.UserException):
      _ops.check_worker_momentum(beta, dampening)
  with pytest.raises(tools.UserException):
    _manager("average", 3, worker_momentum=1.5)
  base = ["--server", "x", "--experiment", "mnist", "--aggregator", "centered-clipping", "--nb-workers", "4"]
  args = runner.make_parser().parse_args(base + ["--worker-momentum", "0.9", "--worker-momentum-dampening", "0.1"])
  assert (args.worker_momentum, args.worker_momentum_dampening) == (0.9, 0.1)
  args = runner.make_parser().parse_args(base)
  assert (args.worker_momentum, args.worker_momentum_dampening) == (0.0, 0.0)


def _manager(gar_name, n, f=0, attack=None, real=0, args=(), **kwargs):
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate(gar_name, n, f, list(args))
  return Manager(experiment, gar, n, "sgd", [], "fixed", ["initial-rate:0.05"], device="cpu", attack=attack, nb_real_byz=real, **kwargs)


def test_switched_off_is_bit_identical_to_no_option():
  plain = _manager("median", 3)
  off = _manager("median", 3, worker_momentum=0.0, worker_momentum_dampening=0.0)
  assert off.worker_momentum is None and not off.momentum_on
  for _ in range(3):
    plain.train()
    off.train()
  _equal_bits(plain.params, off.params)
  assert "worker_momentum" not in off.state_dict()


def test_byzantine_worker_keeps_its_honest_momentum_under_flip():
  beta, c = _ops.check_worker_momentum(0.9, 0.1)
  mgr = _manager("centered-clipping", 5, 1, attacks.instantiate("flip", 5, 1, ["factor:-3"]), 1, worker_momentum=0.9, worker_momentum_dampening=0.1)
  row = mgr.placement[4][1]
  seen = {}
  apply = mgr._apply_momentum

  def recording():
    seen["grad"], seen["momentum"] = mgr.grads[row].clone(), mgr.worker_momentum[row].clone()
    apply()
    seen["after"] = mgr.grads[row].clone()
  mgr._apply_momentum = recording
  for _ in range(3):
    mgr.train()
    expect = torch.add(torch.mul(seen["momentum"], torch.tensor(beta)), torch.mul(seen["grad"], torch.tensor(c)))
    _equal_bits(mgr.worker_momentum[row], expect)   # the honest momentum of the Byzantine worker's own gradient
    _equal_bits(seen["after"], expect)              # what the attack received
    _equal_bits(mgr.grads[row], expect * -3.0)      # what it submitted


def _advance(mgr, steps):
  for stream in mgr.streams:
    for _ in range(steps):
      next(stream)


def test_checkpoint_and_resume_is_bit_identical():
  kwargs = dict(args=["iterations:2", "tau:0.5"], worker_momentum=0.9, worker_momentum_dampening=0.1)
  straight = _manager("centered-clipping", 4, 1, **kwargs)
  for _ in range(4):
    straight.train()
  first = _manager("centered-clipping", 4, 1, **kwargs)
  for _ in range(2):
    first.train()
  state = first.state_dict()
  assert state["worker_momentum"].shape == (4, first.layout.padded_size)
  assert state["aggregation"]["rule_state"].shape == (first.layout.padded_size,)
  resumed = _manager("centered-clipping", 4, 1, **kwargs)
  resumed.load_state_dict(state)
  _advance(resumed, 2)   # the input streams restart with the process: skip the batches the first run consumed
  for _ in range(2):
    resumed.train()
  _equal_bits(resumed.params, straight.params)
  _equal_bits(resumed.worker_momentum, straight.worker_momentum)
  _equal_bits(resumed.aggregation.center, straight.aggregation.center)


def test_checkpoints_without_momenta_or_with_momentum_off(monkeypatch):
  warnings = []
  monkeypatch.setattr(tools, "warning", lambda message, *args, **kwargs: warnings.append(message))
  on = _manager("average", 2, worker_momentum=0.5)
  on.train()
  off = _manager("average", 2)
  off.train()
  on.load_state_dict(off.state_dict())   # an older checkpoint: the momenta restart from zero
  assert not bool(on.worker_momentum.any()) and any("momentum" in w for w in warnings)
  warnings.clear()
  state = _manager("average", 2, worker_momentum=0.5).state_dict()
  off.load_state_dict(state)             # momentum off: the saved momenta are ignored
  assert any("momentum" in w for w in warnings)

"""sm_90a worker momentum: the kernel against the torch reference bit for bit (one and eight rows, d a multiple of 4 or not, strided
rows, NaN and infinities), and the whole-step CUDA graph of a run with worker momentum and centered clipping against an eager run."""

import pytest
import torch

from aggregathor_b200 import aggregators, experiments
from aggregathor_b200.aggregators import _ops
from aggregathor_b200.engine.trainer import Manager
from aggregathor_b200.ops import gar as gar_ops

pytestmark = pytest.mark.gpu


def _equal_bits(a, b):
  a, b = a.cpu(), b.cpu()
  assert a.dtype == b.dtype and a.shape == b.shape
  nan = torch.isnan(a)
  assert torch.equal(nan, torch.isnan(b))
  diff = (a[~nan].view(torch.int32) != b[~nan].view(torch.int32)).nonzero()
  assert diff.numel() == 0, (diff[0].tolist(), float(a[~nan][diff[0]]), float(b[~nan][diff[0]]))


def _rows(w, d, seed):
  gen = torch.Generator().manual_seed(seed)
  G = torch.randn(w, d, generator=gen) * 3
  G[0, 5::97] = float("nan")
  G[-1, 7::89] = float("inf")
  G[-1, 11::83] = float("-inf")
  G[0, 13::79] = 1e38   # beta * M + c * G overflows to infinity after a few steps
  return G


@pytest.mark.parametrize("coefs", [(0.9, 0.0), (0.9, 0.1), (0.5, 0.5), (0.0, 0.3), (0.99, 0.0)])
@pytest.mark.parametrize("d", [400000, 400003])
@pytest.mark.parametrize("w", [1, 8])
def test_kernel_matches_the_torch_reference(w, d, coefs):
  beta, c = _ops.check_worker_momentum(*coefs)
  M_dev = torch.zeros(w, d, device="cuda")
  M_ref = torch.zeros(w, d)
  for step in range(3):
    G = _rows(w, d, seed=step * 7 + w + d)
    G_dev = G.cuda()
    gar_ops.worker_momentum_(G_dev, M_dev, beta, c)
    _ops.torch_worker_momentum_(G, M_ref, beta, c)
    torch.cuda.synchronize()
    _equal_bits(M_dev, M_ref)
    _equal_bits(G_dev, G)


def test_strided_rows():
  """Rows of a wider matrix (the gradient rows of an engine) and unaligned rows take the same values as contiguous ones."""
  w, d = 8, 4099
  beta, c = _ops.check_worker_momentum(0.9, 0.1)
  for width, offset in ((4104, 0), (4100, 1)):
    wide = torch.zeros(w, width + offset, device="cuda")
    M_dev, M_ref = torch.zeros(w, d, device="cuda"), torch.zeros(w, d)
    for step in range(2):
      G = _rows(w, d, seed=step + width)
      view = wide[:, offset:offset + d]
      view.copy_(G)
      gar_ops.worker_momentum_(view, M_dev, beta, c)
      _ops.torch_worker_momentum_(G, M_ref, beta, c)
      torch.cuda.synchronize()
      _equal_bits(M_dev, M_ref)
      _equal_bits(view, G)
      assert not bool(wide[:, :offset].any()) and not bool(wide[:, offset + d:].any())


def _manager(engine, **kwargs):
  experiment = experiments.instantiate("mnist", ["batch-size:16"])
  gar = aggregators.instantiate("centered-clipping", 8, 2, ["iterations:2", "tau:1"])
  return Manager(experiment, gar, 8, "sgd", [], "fixed", ["initial-rate:0.05"], device="cuda", engine=engine, seed=3, **kwargs)


def test_whole_step_graph_equals_eager(monkeypatch):
  graphed = _manager("fused", worker_momentum=0.9, worker_momentum_dampening=0.1)
  for _ in range(5):
    graphed.train()
  torch.cuda.synchronize()
  assert graphed._graph is not None and graphed._graph_whole
  monkeypatch.setenv("AGB_NO_GRAPH", "1")
  eager = _manager("fused", worker_momentum=0.9, worker_momentum_dampening=0.1)
  for _ in range(5):
    eager.train()
  torch.cuda.synchronize()
  assert eager._graph is None
  _equal_bits(graphed.params, eager.params)
  _equal_bits(graphed.worker_momentum, eager.worker_momentum)
  _equal_bits(graphed.aggregation.center, eager.aggregation.center)
  assert bool(graphed.worker_momentum.any())
  graphed.close()
  eager.close()


def test_momentum_off_launches_nothing_new():
  """beta = dampening = 0: no momentum buffer, and the parameters equal those of a run without the options."""
  plain = _manager("fused")
  off = _manager("fused", worker_momentum=0.0, worker_momentum_dampening=0.0)
  assert off.worker_momentum is None and not off.momentum_on
  for _ in range(3):
    plain.train()
    off.train()
  torch.cuda.synchronize()
  _equal_bits(plain.params, off.params)
  plain.close()
  off.close()

"""CUDA graph capture of the training step while other host threads use the GPU.

The input pipelines' producer threads allocate device memory, copy pinned batches on their own streams and synchronise on events
at any time, including while the trainer captures its step graph. The capture must survive that: a capture invalidated by another
thread falls back to eager steps, and leaves torch's default CUDA generator in capture mode, so every later `torch.randn` on the
device in the same process fails."""

import threading

import pytest
import torch

from aggregathor_b200 import aggregators, experiments
from aggregathor_b200.engine.trainer import Manager


def _producer_like_work(device, errors):
  """What a producer thread does for one batch: a fresh device allocation, a pinned host -> device copy on a side stream, an event
  wait."""
  try:
    torch.cuda.set_device(device)
    stream = torch.cuda.Stream(device)
    host = torch.ones(3 << 20, dtype=torch.uint8).pin_memory()
    with torch.cuda.stream(stream):
      dev = host.to(device, non_blocking=True)
      fresh = torch.empty(96 << 20, dtype=torch.uint8, device=device)
      fresh.fill_(1)
      done = torch.cuda.Event()
      done.record(stream)
    done.synchronize()
    assert int(dev[0]) == 1
  except Exception as err:   # noqa: BLE001 - reported by the test thread
    errors.append(err)


@pytest.mark.gpu
def test_capture_survives_another_thread_using_the_gpu(monkeypatch):
  run_workers = Manager._run_workers
  errors, ran = [], []

  def run_workers_with_a_busy_thread(self, *args, **kwargs):
    out = run_workers(self, *args, **kwargs)
    if torch.cuda.is_current_stream_capturing():
      worker = threading.Thread(target=_producer_like_work, args=(self.device, errors))
      worker.start()
      worker.join()
      ran.append(True)
    return out

  monkeypatch.setattr(Manager, "_run_workers", run_workers_with_a_busy_thread)
  gar = aggregators.instantiate("krum", 8, 2, [])
  mgr = Manager(experiments.instantiate("mnist", ["batch-size:16"]), gar, 8, "sgd", [], "fixed", ["initial-rate:0.05"], device="cuda", engine="fused", seed=3)
  try:
    for _ in range(4):
      mgr.train()
    torch.cuda.synchronize()
    assert ran, "the step was never captured"
    assert not errors, errors
    assert mgr._graph is not None, "the capture failed and the trainer fell back to eager steps"
    assert bool(torch.isfinite(mgr.params).all())
    torch.randn(16, device="cuda")   # the default generator left capture mode with the capture
  finally:
    mgr.close()

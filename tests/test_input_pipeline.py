"""Streaming shard reader (native/py_loader) and slim preprocessing (ops/preprocess.py + native/op_nn/preprocess.cu)."""

import numpy as np
import pytest
import torch

from aggregathor_b200.experiments import _data
from aggregathor_b200.ops.preprocess import Preprocessor


def _shards(tmp_path, counts=(50, 51, 52), shape=(8, 8, 3), split="train"):
  rng = np.random.default_rng(0)
  paths = []
  for i, n in enumerate(counts):
    x = rng.integers(0, 255, size=(n,) + shape, dtype=np.uint8)
    y = np.arange(n) + 1000 * i
    x[:, 0, 0, 0] = (y % 251).astype(np.uint8)   # the label is recoverable from the pixels: records stay paired
    paths.append(_data.write_shard(tmp_path / ("%s-%05d-of-%05d.agbshard" % (split, i, len(counts))), x, y))
  return paths


def test_shard_roundtrip_and_header(tmp_path):
  paths = _shards(tmp_path)
  header = _data.read_shard_header(paths[1])
  assert header["count"] == 51 and header["shape"] == (8, 8, 3) and header["record_bytes"] == 192
  x, y = _data.read_shard(paths[1], limit=7)
  assert x.shape == (7, 8, 8, 3) and y.tolist() == list(range(1000, 1007))
  with pytest.raises(Exception):
    _data.read_shard_header(__file__)


def test_shard_stream_covers_the_dataset_and_keeps_pairs(tmp_path):
  paths = _shards(tmp_path)
  stream = _data.ShardStream(paths, 16, "cpu", seed=1, readers=2)
  assert stream.total == 153 and stream.sample_shape == (8, 8, 3)
  seen = []
  for _ in range(40):
    x, y = next(stream)
    assert x.shape == (16, 8, 8, 3) and x.dtype == torch.uint8
    assert torch.equal(x[:, 0, 0, 0].long(), y % 251)
    seen += y.tolist()
  stream.close()
  assert len(set(seen)) >= 150                      # several epochs through a shuffle pool: (almost) everything shows up
  assert seen[:16] != sorted(seen[:16])             # shuffled
  ordered = _data.ShardStream(paths, 10, "cpu", shuffle=False)
  assert next(ordered)[1].tolist() == list(range(10))
  ordered.close()


def test_shard_stream_partitions_are_disjoint(tmp_path):
  paths = _shards(tmp_path)
  a = _data.ShardStream(paths, 8, "cpu", seed=3, readers=2, part=0, parts=2)
  b = _data.ShardStream(paths, 8, "cpu", seed=3, readers=2, part=1, parts=2)
  ya = set(sum([next(a)[1].tolist() for _ in range(25)], []))
  yb = set(sum([next(b)[1].tolist() for _ in range(25)], []))
  a.close(), b.close()
  assert not (ya & yb) and len(ya) > 60 and len(yb) > 60


def test_streamed_dataset_feeds_an_experiment(tmp_path, monkeypatch):
  from aggregathor_b200 import experiments
  from aggregathor_b200.tools import datasets as dataset_tool
  rng = np.random.default_rng(1)
  x = rng.integers(0, 255, size=(200, 40, 40, 3), dtype=np.uint8)
  y = rng.integers(0, 5, size=200)
  dataset_tool.write_shards("tinyset", x[:160], y[:160], x[160:], y[160:], shards=4, output=tmp_path / "tinyset")
  monkeypatch.setenv("AGB_DATASETS", str(tmp_path))
  data = _data.Dataset("tinyset")
  assert data.streaming and data.classes == 5 and data.shape == (40, 40, 3) and data.train_count == 160 and len(data.y_test) == 40
  experiment = experiments.slims.SlimExperiment("tinyset", "lenet", ["batch-size:8", "image-size:28", "nb-fetcher-threads:2"])
  stream = experiment.train_stream(0, 2, "cpu")
  images, labels = next(stream)
  assert images.shape == (8, 40, 40, 3)
  from aggregathor_b200.models import Context
  ctx = Context("torch", True, torch.float32, "cpu")
  out = experiment.preprocess(images, ctx, True)
  assert out.shape == (8, 3, 28, 28) and torch.isfinite(out).all()
  stream.close()


# ---------------------------------------------------------------------------- #
def _images(n=6, size=40, channels=3, seed=0):
  return torch.from_numpy(np.random.default_rng(seed).integers(0, 255, size=(n, size, size, channels), dtype=np.uint8))


def test_vgg_eval_is_a_central_crop_at_matching_resolution():
  pre = Preprocessor("vgg", 24, resize_min=40, resize_max=64)
  x = _images()
  out = pre(x, torch.float32, False)
  expected = x[:, 8:32, 8:32, :].float() - torch.tensor([123.68, 116.78, 103.94])
  assert torch.allclose(out.permute(0, 2, 3, 1), expected, atol=1e-4)


def test_vgg_training_crops_flips_and_replays():
  pre = Preprocessor("vgg", 24, resize_min=40, resize_max=80, seed=5)
  x = _images(64)
  first = pre(x, torch.float32, True, advance=False)
  again = pre(x, torch.float32, True, advance=True)
  assert torch.equal(first, again)                      # same counter -> same augmentation
  later = pre(x, torch.float32, True)
  assert not torch.equal(first, later)                  # advanced counter -> new draws
  params = pre.sampling(64, 40, 40, True, 0)
  assert 10 < int(params["flip"].sum()) < 54
  assert (params["y0"] >= 0).all() and (params["y0"] + 24 * params["sy"] <= 40 + 1e-3).all()
  other = pre(x, torch.float32, True, advance=False, stream_id=3)
  assert not torch.equal(other, pre(x, torch.float32, True, advance=False))


def test_cifarnet_standardises_and_matches_the_plain_formula_in_eval():
  pre = Preprocessor("cifarnet", 32, pad=4)
  x = _images(5, 32)
  out = pre(x, torch.float32, False)
  flat = x.float().reshape(5, -1)
  expected = (x.float() - flat.mean(1).view(5, 1, 1, 1)) / torch.clamp(flat.std(1, unbiased=False), min=1.0 / (32 * 32 * 3) ** 0.5).view(5, 1, 1, 1)
  assert torch.allclose(out.permute(0, 2, 3, 1), expected, atol=1e-3)
  train = pre(x, torch.float32, True)
  assert torch.allclose(train.mean(dim=(1, 2, 3)), torch.zeros(5), atol=1e-3) and torch.allclose(train.flatten(1).std(1, unbiased=False), torch.ones(5), atol=1e-2)


def test_inception_ranges():
  pre = Preprocessor("inception", 20, seed=2)
  x = _images(32, 48)
  out = pre(x, torch.float32, True)
  assert out.shape == (32, 3, 20, 20) and float(out.min()) >= -1.0 and float(out.max()) <= 1.0
  params = pre.sampling(32, 48, 48, True, 0)
  box_w, box_h = params["sx"] * 20, params["sy"] * 20
  assert (box_w <= 48 + 1e-3).all() and (box_h <= 48 + 1e-3).all() and set(np.unique(params["ordering"])) <= {0, 1, 2, 3}
  aspect = box_w / box_h
  assert (aspect > 0.74).all() and (aspect < 1.34).all()
  ev = pre(x, torch.float32, False)
  assert ev.shape == (32, 3, 20, 20)


@pytest.mark.gpu
@pytest.mark.parametrize("mode,size,store,training", [("vgg", 224, 256, True), ("vgg", 224, 256, False), ("inception", 299, 320, True), ("inception", 224, 256, False),
                                                       ("cifarnet", 32, 32, True), ("cifarnet", 32, 32, False), ("plain", 28, 28, False)])
def test_preprocess_kernel_matches_the_torch_arithmetic(mode, size, store, training):
  channels = 1 if mode == "plain" else 3
  x = _images(16, store, channels, seed=3).cuda()
  kwargs = dict(mean=(128.0, 128.0, 128.0), scale=1 / 128.0) if mode == "plain" else {}
  pre = Preprocessor(mode, size, seed=11, **kwargs)
  pre.counter("cuda").fill_(7)
  native = pre(x, torch.float32, training, backend="native", advance=False)
  reference = pre._torch(x, torch.float32, training, 7, pre.seed)
  assert native.shape == reference.shape
  diff = (native - reference).abs()
  scale = float(reference.abs().max())
  # Every pixel, no outlier allowance: bilinear sampling is continuous in its coordinate, so the rounding differences between the
  # two sides (contracted multiply-adds, summation order) move a value by a few fp32 ulps of the coordinate times 255, far below
  # this bound, and a differing discrete decision (crop floor, box acceptance) would move a whole image, not scattered pixels.
  # No pixel needed an allowance at these seeds, and one would hide a defect confined to a border row or column.
  assert float(diff.max()) <= 2e-3 * max(scale, 1.0), float(diff.max())
  bf16 = pre(x, torch.bfloat16, training, backend="native", advance=False)
  assert bf16.dtype == torch.bfloat16 and float((bf16.float() - native).abs().max()) <= 0.01 * max(scale, 1.0) + 1e-2


@pytest.mark.gpu
def test_augmentation_replays_from_a_cuda_graph():
  pre = Preprocessor("cifarnet", 32, seed=1)
  x = _images(8, 32).cuda()
  pre(x, torch.float32, True, backend="native")   # warm-up (lazy module load)
  torch.cuda.synchronize()
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph):
    out = pre(x, torch.float32, True, backend="native")
  graph.replay()
  first = out.clone()
  graph.replay()
  assert not torch.equal(first, out)   # the captured counter increment makes every replay draw new crops


def test_producer_failures_reach_the_consumer():
  """A producer thread that dies hands its exception to `next()` instead of leaving the consumer blocked on an empty queue."""
  import queue
  import threading

  class Failing:
    def __init__(self):
      self._queue, self._stop, self._error = queue.Queue(maxsize=2), False, None

    @_data._guarded
    def _producer(self):
      raise ValueError("no such device")

  stream = Failing()
  threading.Thread(target=stream._producer, daemon=True).start()
  for _ in range(2):
    with pytest.raises(RuntimeError, match="producer thread failed"):
      _data._take(stream)
  assert str(_data._indexed("cpu")) == "cpu"


@pytest.mark.gpu
def test_stream_group_serves_every_worker_its_own_sequence():
  """`StreamGroup`: one producer / pinned slab / H2D copy per step for all the workers of a rank; every worker still receives exactly
  the batches its own `BatchStream` (same seed) would have produced, as slices of one device tensor."""
  rng = np.random.default_rng(0)
  images = rng.integers(0, 255, size=(96, 6, 5, 3), dtype=np.uint8)
  labels = np.arange(96, dtype=np.int64)
  make = lambda seed, transform=None: _data.BatchStream(images, labels, 8, "cuda", seed=seed, transform=transform)
  group = _data.StreamGroup([make(1), make(2), make(3)])
  reference = [make(1), make(2), make(3)]
  assert _data.StreamGroup.eligible(group.streams) and not _data.StreamGroup.eligible([reference[0], reference[0]])
  for _ in range(15):                      # crosses an epoch boundary (96 / 8 = 12 batches)
    batches = next(group)
    assert isinstance(batches, _data.GroupedBatches) and batches.x_all.shape == (3, 8, 6, 5, 3) and batches.y_all.shape == (3, 8)
    for (x, y), source in zip(batches, reference):
      want_x, want_y = next(source)
      assert torch.equal(x, want_x) and torch.equal(y, want_y)
      assert torch.equal(x.cpu(), torch.from_numpy(images[y.cpu().numpy()]))
  shifted = _data.StreamGroup([make(1, lambda x, y: (x, y - 1)), make(2, lambda x, y: (x, y - 1))])
  batches = next(shifted)
  assert batches.x_all is not None and batches.y_all is None and int(batches[0][1].min()) >= -1
  for s in (group, shifted):
    s.close()
  for s in reference:
    s.close()

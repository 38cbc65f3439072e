"""The Dirichlet label partition (`dirichlet:<alpha>`) on the CPU: the partition's invariants and fixed algorithm, label concentration as
alpha varies, the argument checks, the unchanged streams without it, and the native shard reader's subsets."""

import numpy as np
import pytest

from aggregathor_b200 import experiments, tools
from aggregathor_b200.experiments import _data


def _labels():
  return experiments.instantiate("mnist", ["batch-size:16"]).data.y_train


def _pinned(labels, n, alpha, seed, min_size):
  """The algorithm as specified, written out once more: per class, permute, draw p, cut at floor(cumsum(p)[:-1] * count)."""
  rng = np.random.default_rng([seed, 0x4449524C])
  while True:
    parts = [[] for _ in range(n)]
    for c in np.unique(labels):
      members = rng.permutation(np.flatnonzero(labels == c))
      p = rng.dirichlet([alpha] * n)
      cuts = [0] + [int(x) for x in np.floor(np.cumsum(p)[:-1] * len(members))] + [len(members)]
      for i in range(n):
        parts[i].extend(members[cuts[i]:cuts[i + 1]].tolist())
    if min(len(p) for p in parts) >= min_size:
      return [np.array(sorted(p), dtype=np.int64) for p in parts]


@pytest.mark.parametrize("n,alpha,seed", [(8, 0.3, 0), (5, 1.0, 7), (16, 100.0, 3)])
def test_partition_is_disjoint_covering_and_pinned(n, alpha, seed):
  labels = _labels()
  parts = _data.dirichlet_partition(labels, n, alpha, seed, 16)
  assert len(parts) == n
  assert all(p.dtype == np.int64 and np.all(np.diff(p) > 0) and len(p) >= 16 for p in parts)
  joined = np.concatenate(parts)
  assert len(joined) == len(labels) and np.array_equal(np.sort(joined), np.arange(len(labels)))
  expected = _pinned(labels, n, alpha, seed, 16)
  assert all(np.array_equal(a, b) for a, b in zip(parts, expected))
  again = _data.dirichlet_partition(labels, n, alpha, seed, 16)
  assert all(np.array_equal(a, b) for a, b in zip(parts, again))
  other = _data.dirichlet_partition(labels, n, alpha, seed + 1, 16)
  assert any(not np.array_equal(a, b) for a, b in zip(parts, other))


def _concentration(labels, parts, classes):
  """Mean over workers of the share of the worker's most frequent class."""
  return float(np.mean([np.bincount(labels[p], minlength=classes).max() / len(p) for p in parts]))


def test_alpha_controls_label_skew():
  labels = _labels()
  skewed = _data.dirichlet_partition(labels, 10, 0.1, 1, 16)
  uniform = _data.dirichlet_partition(labels, 10, 1000.0, 1, 16)
  iid_share = np.bincount(labels).max() / len(labels)
  assert _concentration(labels, skewed, 10) > 0.5
  assert abs(_concentration(labels, uniform, 10) - iid_share) < 0.03
  assert min(len(np.unique(labels[p])) for p in uniform) == 10
  sizes = [len(p) for p in uniform]
  assert max(sizes) - min(sizes) < 0.1 * len(labels) / 10


def test_infeasible_sizes_and_bad_arguments_raise():
  labels = _labels()
  with pytest.raises(tools.UserException, match="n = 64"):
    _data.dirichlet_partition(labels, 64, 0.01, 0, 256)
  for alpha in ("0", "-1", "inf", "nan", "x"):
    with pytest.raises(tools.UserException):
      experiments.instantiate("mnist", ["dirichlet:" + alpha])
  with pytest.raises(tools.UserException, match="shared-batch"):
    experiments.instantiate("mnist", ["dirichlet:0.5", "shared-batch:1"])
  with pytest.raises(tools.UserException):
    experiments.instantiate("cnnet", ["dirichlet:0"])


def test_streams_without_dirichlet_are_unchanged():
  plain = experiments.instantiate("mnist", ["batch-size:8", "seed:4"])
  data = plain.data
  for worker in range(3):
    stream = plain.train_stream(worker, 3, "cpu")
    rng = np.random.default_rng(4 + worker)
    order = np.arange(len(data.y_train))
    rng.shuffle(order)
    for b in range(2):
      x, y = next(stream)
      idx = order[b * 8:(b + 1) * 8]
      assert np.array_equal(y.numpy(), data.y_train[idx]) and np.array_equal(x.numpy(), data.x_train[idx])


def test_worker_streams_draw_from_their_part_only():
  exp = experiments.instantiate("mnist", ["batch-size:8", "dirichlet:0.3", "seed:2"])
  parts = _data.dirichlet_partition(exp.data.y_train, 4, 0.3, 2, 8)
  images = exp.data.x_train.reshape(len(exp.data.x_train), -1)
  for worker in range(4):
    stream = exp.train_stream(worker, 4, "cpu")
    assert stream.images is exp.data.x_train   # no copy of the images
    seen = set()
    for _ in range(-(-len(parts[worker]) // 8)):
      x, y = next(stream)
      rows = x.numpy().reshape(8, -1)
      for row, label in zip(rows, y.numpy()):
        matches = np.flatnonzero((images[parts[worker]] == row).all(axis=1))
        assert len(matches) >= 1 and exp.data.y_train[parts[worker][matches[0]]] == label
        seen.update(parts[worker][matches].tolist())
    assert len(seen) >= len(parts[worker]) - 8   # the first epoch serves every sample but the remainder of the last batch
  stream = exp.train_stream(0, 4, "cpu")
  assert _data.StreamGroup.eligible([stream]) is False   # one stream: not a group, but a plain BatchStream
  assert type(stream) is _data.BatchStream


# ---------------------------------------------------------------------------- #
# Streamed datasets: the native reader serves a membership bitmap over the global record index

def _shards(tmp_path, counts=(50, 51, 52), shape=(8, 8, 3), classes=5):
  rng = np.random.default_rng(0)
  paths, first = [], 0
  for i, n in enumerate(counts):
    x = rng.integers(0, 255, size=(n,) + shape, dtype=np.uint8)
    ids = np.arange(first, first + n)
    x[:, 0, 0, 0] = (ids % 251).astype(np.uint8)   # the global record index is recoverable from the pixels
    x[:, 0, 0, 1] = (ids // 251).astype(np.uint8)
    paths.append(_data.write_shard(tmp_path / ("train-%05d-of-%05d.agbshard" % (i, len(counts))), x, ids % classes))
    first += n
  return paths


def _ids(x):
  return (x[:, 0, 0, 0].long() + 251 * x[:, 0, 0, 1].long()).tolist()


def test_shard_subset_serves_exactly_its_records_in_one_epoch(tmp_path):
  """Sequential order: one epoch of the subset reader is its records, ascending, each once."""
  paths = _shards(tmp_path)
  labels = np.arange(153) % 5
  subset = np.sort(np.random.default_rng(4).choice(153, size=48, replace=False))
  stream = _data.ShardStream(paths, 8, "cpu", shuffle=False, subset=subset)
  assert stream.total == 48
  seen = []
  for _ in range(6):   # one epoch: 48 records
    x, y = next(stream)
    ids = _ids(x)
    assert y.tolist() == labels[ids].tolist()
    seen += ids
  assert seen == subset.tolist()
  assert _ids(next(stream)[0]) == subset[:8].tolist()   # the next epoch starts over
  stream.close()


def test_shuffled_shard_subset_stays_inside_its_records(tmp_path):
  """Several readers and a shuffle pool (which may already hold the next epoch's records): only subset records, (almost) all of them."""
  paths = _shards(tmp_path)
  subset = np.sort(np.random.default_rng(5).choice(153, size=48, replace=False))
  stream = _data.ShardStream(paths, 8, "cpu", seed=2, readers=2, subset=subset)
  seen = []
  for _ in range(18):   # three epochs
    seen += _ids(next(stream)[0])
  stream.close()
  assert set(seen) <= set(subset.tolist())
  assert len(set(seen)) >= 44   # uniform draws from the pool: a record may wait there past the epoch
  assert seen[:8] != sorted(seen[:8])


def test_shard_subset_rejects_bad_bitmaps(tmp_path):
  paths = _shards(tmp_path)
  with pytest.raises(tools.UserException):
    _data.ShardStream(paths, 8, "cpu", subset=np.array([], dtype=np.int64))
  with pytest.raises(tools.UserException):
    _data.ShardStream(paths, 8, "cpu", subset=np.array([153]))


def test_streamed_dataset_partitions_from_its_shard_labels(tmp_path, monkeypatch):
  from aggregathor_b200.tools import datasets as dataset_tool
  rng = np.random.default_rng(1)
  x = rng.integers(0, 255, size=(200, 40, 40, 3), dtype=np.uint8)
  y = rng.integers(0, 5, size=200)
  dataset_tool.write_shards("tinyset", x[:160], y[:160], x[160:], y[160:], shards=4, output=tmp_path / "tinyset")
  monkeypatch.setenv("AGB_DATASETS", str(tmp_path))
  experiment = experiments.slims.SlimExperiment("tinyset", "lenet", ["batch-size:8", "image-size:28", "dirichlet:0.5", "seed:3"])
  data = experiment.data
  assert data.streaming
  shard_labels = np.concatenate([_data.read_shard(p)[1] for p in data.train_shards])
  assert np.array_equal(data.train_labels(), shard_labels)
  parts = _data.dirichlet_partition(shard_labels, 2, 0.5, 3, 8)
  images = np.concatenate([_data.read_shard(p)[0] for p in data.train_shards]).reshape(160, -1)
  for worker in range(2):
    stream = experiment.train_stream(worker, 2, "cpu")
    assert stream.total == len(parts[worker])
    got = np.asarray(next(stream)[0]).reshape(8, -1)
    for row in got:
      assert (images[parts[worker]] == row).all(axis=1).any()
    stream.close()

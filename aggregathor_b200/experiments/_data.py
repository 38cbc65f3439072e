"""Datasets: on-disk loaders when the files exist, deterministic synthetic stand-ins otherwise.

The reference reads MNIST through `tf.keras.datasets.mnist.load_data()` and CIFAR-10 / ImageNet TFRecords through
slim from user-provided `experiments/datasets/<name>` directories (`README.md:190-195`). This sandbox has no network
and no datasets, so every dataset has a *synthetic* twin of the same shape and dtype: class-conditional prototypes
plus noise (learnable, so the training loop still shows a falling loss / rising accuracy). Real data is picked up from
`experiments/datasets/<name>/` (`.npz` with `x_train,y_train,x_test,y_test`, uint8 NHWC) or `$AGB_DATASETS/<name>/`.

`BatchStream` is the input pipeline: a background thread assembles batches into pinned host buffers and issues the
host->device copies on a side stream, double-buffered, so the step never waits on the input unless it outruns it.

Datasets that do not fit in host memory (ImageNet at 256x256 is ~250 GB) are *streamed*: `tools/datasets.py --shards N` writes
`<name>/train-00000-of-000NN.agbshard` files of fixed-size records and `ShardStream` feeds the same pinned ring from the native
reader (`native/py_loader`: reader threads -> shuffle pool -> batch), the counterpart of slim's `DatasetDataProvider(num_readers)`
+ `tf.train.batch` + `prefetch_queue` (reference: `experiments/slims.py:100-111`, `experiments/cnnet.py:123-132`).
"""

import ctypes
import json
import os
import pathlib
import queue
import struct
import threading

import numpy as np
import torch

from .. import tools

DATASETS_DIR = pathlib.Path(__file__).parent / "datasets"

_SHAPES = {  # name -> (train size, test size, (H, W, C), classes)
  "mnist": (60000, 10000, (28, 28, 1), 10),
  "cifar10": (50000, 10000, (32, 32, 3), 10),
  "cifar100": (50000, 10000, (32, 32, 3), 100),
  "flowers": (3320, 350, (224, 224, 3), 5),
  "imagenet": (1281167, 50000, (224, 224, 3), 1000)}


SHARD_MAGIC = b"AGBSHRD1"
SHARD_SUFFIX = ".agbshard"


def write_shard(path, images, labels):
  """One shard file: 64-byte header, `count` uint8 HWC records, `count` int64 labels (layout of `native/py_loader/loader.cpp`)."""
  images = np.ascontiguousarray(images, dtype=np.uint8)
  labels = np.ascontiguousarray(labels, dtype=np.int64).reshape(-1)
  if images.ndim == 3:
    images = images[..., None]
  count, h, w, c = images.shape
  if len(labels) != count:
    raise tools.UserException("write_shard: %d images but %d labels" % (count, len(labels)))
  header = SHARD_MAGIC + struct.pack("<QIIIIQ", count, h, w, c, 8, h * w * c) + bytes(24)
  with open(path, "wb") as fd:
    fd.write(header)
    fd.write(images.tobytes())
    fd.write(labels.tobytes())
  return path


def read_shard_header(path):
  with open(path, "rb") as fd:
    raw = fd.read(64)
  if len(raw) != 64 or raw[:8] != SHARD_MAGIC:
    raise tools.UserException("Not a shard file: " + repr(str(path)))
  count, h, w, c, label_bytes, record_bytes = struct.unpack("<QIIIIQ", raw[8:40])
  return {"count": count, "shape": (h, w, c), "record_bytes": record_bytes, "label_bytes": label_bytes}


def read_shard(path, limit=None):
  """Whole shard (or its first `limit` records) in memory: the evaluation split, tests."""
  header = read_shard_header(path)
  count = header["count"] if limit is None else min(header["count"], limit)
  with open(path, "rb") as fd:
    fd.seek(64)
    images = np.frombuffer(fd.read(count * header["record_bytes"]), dtype=np.uint8).reshape((count,) + header["shape"])
    fd.seek(64 + header["count"] * header["record_bytes"])
    labels = np.frombuffer(fd.read(count * 8), dtype=np.int64)
  return images, labels


def _dataset_roots():
  return (DATASETS_DIR, pathlib.Path(os.environ.get("AGB_DATASETS", "/nonexistent")))


def find_shards(name, split):
  """Sorted shard files `<root>/<name>/<split>-*.agbshard` of a streamed dataset ([] when there are none)."""
  for root in _dataset_roots():
    files = sorted((root / name).glob(split + "-*" + SHARD_SUFFIX)) if (root / name).is_dir() else []
    if files:
      return files
  return []


def known_datasets():
  names = dict(_SHAPES)
  for root in (DATASETS_DIR, pathlib.Path(os.environ.get("AGB_DATASETS", "/nonexistent"))):
    if root.is_dir():
      for path in root.iterdir():
        if path.is_dir() and path.name not in names and tools.can_access(path, read=True):
          names[path.name] = None
  return names


def _find_npz(name):
  for root in (DATASETS_DIR, pathlib.Path(os.environ.get("AGB_DATASETS", "/nonexistent")), pathlib.Path.home() / ".keras" / "datasets"):
    for candidate in (root / name / (name + ".npz"), root / (name + ".npz")):
      if candidate.is_file():
        return candidate
  return None


class Dataset:
  """In-memory (or lazily synthesised) classification dataset: uint8 NHWC images + int64 labels."""

  def __init__(self, name, image_size=None, synthetic_limit=4096, seed=1234):
    self.name = name
    self.streaming = False
    self.train_shards = find_shards(name, "train")
    if self.train_shards:
      # streamed dataset: only the (bounded) evaluation split is held in memory
      self.streaming, self.synthetic = True, False
      header = read_shard_header(self.train_shards[0])
      self.shape = header["shape"]
      self.train_count = sum(read_shard_header(p)["count"] for p in self.train_shards)
      test_shards = find_shards(name, "test") or find_shards(name, "validation")
      parts = [read_shard(p, limit=4096) for p in test_shards[:4]] or [read_shard(self.train_shards[-1], limit=1024)]
      self.x_test, self.y_test = np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
      self.x_train, self.y_train = None, None
      meta = self.train_shards[0].parent / "meta.json"
      if meta.is_file():
        self.classes = int(json.loads(meta.read_text())["classes"])
      else:
        self.classes = int(max(int(read_shard(p)[1].max()) for p in self.train_shards)) + 1
      return
    path = _find_npz(name)
    if path is not None:
      with np.load(path) as blob:
        self.x_train, self.y_train = blob["x_train"], blob["y_train"].astype(np.int64).reshape(-1)
        self.x_test, self.y_test = blob["x_test"], blob["y_test"].astype(np.int64).reshape(-1)
      if self.x_train.ndim == 3:
        self.x_train, self.x_test = self.x_train[..., None], self.x_test[..., None]
      self.synthetic = False
      self.classes = int(self.y_train.max()) + 1
      self.shape = tuple(self.x_train.shape[1:])
      self.train_count = len(self.y_train)
      return
    if name not in _SHAPES or _SHAPES[name] is None:
      raise tools.UserException("Dataset " + repr(name) + " not found (expected " + repr(str(DATASETS_DIR / name / (name + ".npz"))) + ")")
    ntrain, ntest, shape, classes = _SHAPES[name]
    if image_size is not None:
      shape = (image_size, image_size, shape[2])
    self.synthetic, self.classes, self.shape = True, classes, shape
    rng = np.random.default_rng(seed)
    # low-resolution class prototypes, upsampled: cheap to store, still linearly separable
    low = max(4, min(8, shape[0] // 4))
    self._protos = rng.integers(32, 224, size=(classes, low, low, shape[2]), dtype=np.uint8)
    ntrain, ntest = min(ntrain, synthetic_limit), min(ntest, max(256, synthetic_limit // 4))
    self.y_train = rng.integers(0, classes, size=ntrain, dtype=np.int64)
    self.y_test = rng.integers(0, classes, size=ntest, dtype=np.int64)
    self.x_train = self._render(self.y_train, rng)
    self.x_test = self._render(self.y_test, rng)
    self.train_count = ntrain

  def train_stream(self, batch_size, device, seed=0, transform=None, readers=1, part=0, parts=1, indices=None):
    """The training input pipeline of one worker: in-memory `BatchStream`, or the native shard reader when the dataset is streamed
    (`readers` = reader threads, the reference's `nb-fetcher-threads`; `part`/`parts` give each worker a disjoint residue class).
    `indices`: the worker's own training samples (a `dirichlet_partition` part of `train_labels()`), which replace `part`/`parts`."""
    if self.streaming:
      return ShardStream(self.train_shards, batch_size, device, seed=seed, transform=transform, readers=readers, part=part, parts=parts, subset=indices)
    return BatchStream(self.x_train, self.y_train, batch_size, device, seed=seed, transform=transform, indices=indices)

  def train_labels(self):
    """The labels of the training set by global record index: in memory, or read from the label section of every shard, in the sorted
    order of the shard files (no image is read)."""
    if not self.streaming:
      return self.y_train
    if getattr(self, "_shard_labels", None) is None:
      parts = []
      for path in self.train_shards:
        header = read_shard_header(path)
        with open(path, "rb") as fd:
          fd.seek(64 + header["count"] * header["record_bytes"])
          parts.append(np.frombuffer(fd.read(header["count"] * 8), dtype=np.int64))
      self._shard_labels = np.concatenate(parts)
    return self._shard_labels

  def _render(self, labels, rng):
    h, w, c = self.shape
    low = self._protos.shape[1]
    reps_h, reps_w = -(-h // low), -(-w // low)
    out = np.empty((len(labels), h, w, c), dtype=np.uint8)
    for start in range(0, len(labels), 512):
      chunk = labels[start:start + 512]
      imgs = np.repeat(np.repeat(self._protos[chunk], reps_h, axis=1), reps_w, axis=2)[:, :h, :w, :].astype(np.int16)
      imgs += rng.integers(-48, 48, size=imgs.shape, dtype=np.int16)
      out[start:start + 512] = np.clip(imgs, 0, 255).astype(np.uint8)
    return out


def _indexed(device):
  """`torch.device` with an explicit index for CUDA ("cuda" -> the current device): producer threads call `torch.cuda.set_device`."""
  device = torch.device(device)
  if device.type == "cuda" and device.index is None:
    device = torch.device("cuda", torch.cuda.current_device())
  return device


def _guarded(producer):
  """Producer-thread body that hands its exception to the consumer (a `None` in the queue) instead of dying silently and leaving
  `next()` blocked forever."""
  def run(self):
    try:
      producer(self)
    except BaseException as err:   # noqa: B902 - re-raised in the consumer thread
      self._error = err
      while not self._stop:
        try:
          self._queue.put(None, timeout=0.1)
          break
        except queue.Full:
          continue
  return run


def _stop_producer(self):
  """Stops the producer thread and waits for it (it checks `_stop` at least every 0.1 s): a daemon thread still inside torch when
  the interpreter exits is torn down mid-call, which aborts the process."""
  self._stop = True
  thread = self._thread
  if thread is not None and thread is not threading.current_thread():
    thread.join(timeout=30)


def _take(self):
  item = self._queue.get()
  if item is None:
    self._queue.put(None)          # every later call fails too
    raise RuntimeError("the input pipeline's producer thread failed: %r" % (self._error,)) from self._error
  return item


DIRICHLET_TAG = 0x4449524C   # "DIRL": second word of the partition's generator seed
DIRICHLET_ATTEMPTS = 100


def check_dirichlet(alpha):
  """The concentration of `dirichlet:<alpha>`: a finite float > 0."""
  try:
    value = float(alpha)
  except (TypeError, ValueError):
    raise tools.UserException("dirichlet: expected a number (got %r)" % (alpha,))
  if not np.isfinite(value) or value <= 0:
    raise tools.UserException("dirichlet: alpha must be finite and > 0 (got %r)" % (alpha,))
  return value


def dirichlet_partition(labels, n, alpha, seed, min_size):
  """Label-skewed split of a training set over n workers (Hsu, Qi & Brown, 2019): n sorted, disjoint int64 index arrays whose union is
  every sample. With rng = numpy's default_rng([seed, DIRICHLET_TAG]), for each class c in ascending order: the ascending indices of class
  c are permuted by rng.permutation, p = rng.dirichlet([alpha] * n) is drawn and the permuted indices are cut at floor(cumsum(p)[:-1] *
  count); worker i gets slice i. While a worker gets fewer than `min_size` samples, the whole partition is drawn again from the same rng,
  at most DIRICHLET_ATTEMPTS times in all. Small alpha concentrates every class on few workers; large alpha approaches an IID split."""
  labels = np.asarray(labels).reshape(-1)
  n, alpha, min_size = int(n), check_dirichlet(alpha), int(min_size)
  if n < 1:
    raise tools.UserException("dirichlet: needs at least one worker (got %d)" % n)
  rng = np.random.default_rng([int(seed), DIRICHLET_TAG])
  classes = np.unique(labels)
  for _ in range(DIRICHLET_ATTEMPTS):
    parts = [[] for _ in range(n)]
    for c in classes:
      members = rng.permutation(np.flatnonzero(labels == c))
      p = rng.dirichlet([alpha] * n)
      cuts = np.floor(np.cumsum(p)[:-1] * len(members)).astype(np.int64)
      for i, piece in enumerate(np.split(members, cuts)):
        parts[i].append(piece)
    parts = [np.sort(np.concatenate(piece)).astype(np.int64) for piece in parts]
    if min(len(part) for part in parts) >= min_size:
      return parts
  raise tools.UserException("dirichlet: no partition of the %d samples over n = %d workers with alpha = %g gives every worker a batch of %d "
                            "samples in %d draws" % (len(labels), n, alpha, min_size, DIRICHLET_ATTEMPTS))


class BatchStream:
  """Infinite shuffled batch iterator with pinned double buffering and asynchronous H2D copies. `indices` (optional) restricts the stream
  to those samples (its order before the first shuffle replaces `arange(len(labels))`); no image is copied."""

  def __init__(self, images, labels, batch_size, device, seed=0, shuffle=True, depth=2, transform=None, indices=None):
    self.images, self.labels, self.batch = images, labels, int(batch_size)
    self.device = _indexed(device)
    self.shuffle, self.transform = shuffle, transform
    self._rng = np.random.default_rng(seed)
    self._order = np.arange(len(labels)) if indices is None else np.array(indices, dtype=np.int64)
    self._cursor = len(self._order)  # forces a shuffle at first use
    self._cuda = self.device.type == "cuda"
    self._depth = depth
    self._queue = None
    self._thread = None
    self._stop = False
    self._error = None
    self._lock = threading.Lock()
    self.sample_shape = tuple(images.shape[1:])
    self.sample_dtype = torch.from_numpy(images[:1]).dtype
    self.h2d_bytes = self.batch * int(np.prod(self.sample_shape)) * images.dtype.itemsize + self.batch * 8

  def _next_indices(self):
    with self._lock:   # the stream's own producer thread and a `StreamGroup` may both draw from it
      if self._cursor + self.batch > len(self._order):
        if self.shuffle:
          self._rng.shuffle(self._order)
        self._cursor = 0
      idx = self._order[self._cursor:self._cursor + self.batch].copy()
      self._cursor += self.batch
    return np.sort(idx) if not self.shuffle else idx

  def _host_batch(self, slot=None):
    idx = self._next_indices()
    x = torch.from_numpy(self.images[idx])
    y = torch.from_numpy(self.labels[idx])
    if slot is not None:
      slot[0].copy_(x)
      slot[1].copy_(y)
      return slot
    return x, y

  @_guarded
  def _producer(self):
    torch.cuda.set_device(self.device)
    stream = torch.cuda.Stream(self.device)
    shape = (self.batch,) + self.sample_shape
    slots = [(torch.empty(shape, dtype=self.sample_dtype).pin_memory(), torch.empty(self.batch, dtype=torch.int64).pin_memory()) for _ in range(self._depth + 2)]
    i = 0
    events = [None] * len(slots)
    while not self._stop:
      if events[i % len(slots)] is not None:
        events[i % len(slots)].synchronize()  # the previous copy out of this pinned slot has completed
      host = self._host_batch(slots[i % len(slots)])
      with torch.cuda.stream(stream):
        x = host[0].to(self.device, non_blocking=True)
        y = host[1].to(self.device, non_blocking=True)
        done = torch.cuda.Event()
        done.record(stream)
      events[i % len(slots)] = done
      while not self._stop:
        try:
          self._queue.put((x, y, done), timeout=0.1)
          break
        except queue.Full:
          continue
      i += 1

  def __iter__(self):
    return self

  def __next__(self):
    if not self._cuda:
      x, y = self._host_batch()
      x, y = x.clone(), y.clone()
    else:
      if self._thread is None:
        self._queue = queue.Queue(maxsize=self._depth)
        self._thread = threading.Thread(target=self._producer, name="input", daemon=True)
        self._thread.start()
      x, y, done = _take(self)
      consumer = torch.cuda.current_stream(self.device)
      consumer.wait_event(done)
      # allocated on the producer's side stream, consumed here: tell the caching allocator, or the block could be handed back to the
      # producer's next H2D copy while kernels of this stream still read it
      x.record_stream(consumer)
      y.record_stream(consumer)
    return (x, y) if self.transform is None else self.transform(x, y)

  def close(self):
    _stop_producer(self)


class GroupedBatches(list):
  """The per-worker batches of one step, `[(x, y), ...]`, when they are slices of ONE device tensor each (`x_all`, `y_all`): the
  trainer then refreshes its static graph inputs with one copy instead of one per worker."""
  x_all = None
  y_all = None


class StreamGroup:
  """The in-memory batch streams of the logical workers hosted by one rank, served by ONE producer thread, ONE pinned slab and ONE
  host -> device copy per step (the streams keep their own shuffled orders: every worker still draws its own batches). With `w`
  workers per rank this replaces `w` queues, `2 w` copies and `w` events per step — host work that sits between two steps when the
  caller reads the loss every step."""

  def __init__(self, streams, depth=2):
    self.streams = list(streams)
    first = self.streams[0]
    self.device, self.batch = first.device, first.batch
    self._depth = depth
    self._queue = None
    self._thread = None
    self._stop = False
    self._error = None

  @staticmethod
  def eligible(streams):
    """Plain `BatchStream`s (not the shard reader) of one CUDA device with identical batch geometry, none of them started yet."""
    if len(streams) < 2 or any(type(s) is not BatchStream for s in streams) or len(set(id(s) for s in streams)) != len(streams):
      return False   # (a stream shared by several workers — `shared-batch` — must keep handing out ONE sequence of batches)
    first = streams[0]
    return first._cuda and all(s.device == first.device and s.batch == first.batch and s.sample_shape == first.sample_shape and s.sample_dtype == first.sample_dtype
                               and s._thread is None for s in streams)

  @_guarded
  def _producer(self):
    torch.cuda.set_device(self.device)
    stream = torch.cuda.Stream(self.device)
    first, count = self.streams[0], len(self.streams)
    shape = (count, self.batch) + first.sample_shape
    slots = [(torch.empty(shape, dtype=first.sample_dtype).pin_memory(), torch.empty((count, self.batch), dtype=torch.int64).pin_memory()) for _ in range(self._depth + 2)]
    events = [None] * len(slots)
    i = 0
    while not self._stop:
      slot = slots[i % len(slots)]
      if events[i % len(slots)] is not None:
        events[i % len(slots)].synchronize()  # the previous copy out of this pinned slot has completed
      for j, source in enumerate(self.streams):
        source._host_batch((slot[0][j], slot[1][j]))
      with torch.cuda.stream(stream):
        x = slot[0].to(self.device, non_blocking=True)
        y = slot[1].to(self.device, non_blocking=True)
        done = torch.cuda.Event()
        done.record(stream)
      events[i % len(slots)] = done
      while not self._stop:
        try:
          self._queue.put((x, y, done), timeout=0.1)
          break
        except queue.Full:
          continue
      i += 1

  def __iter__(self):
    return self

  def __next__(self):
    if self._thread is None:
      self._queue = queue.Queue(maxsize=self._depth)
      self._thread = threading.Thread(target=self._producer, name="input-group", daemon=True)
      self._thread.start()
    x, y, done = _take(self)
    consumer = torch.cuda.current_stream(self.device)
    consumer.wait_event(done)
    x.record_stream(consumer)
    y.record_stream(consumer)
    batches = GroupedBatches()
    for j, source in enumerate(self.streams):
      batches.append((x[j], y[j]) if source.transform is None else source.transform(x[j], y[j]))
    batches.x_all = x if all(b[0].data_ptr() == x[j].data_ptr() and b[0].shape == x[j].shape for j, b in enumerate(batches)) else None
    batches.y_all = y if all(b[1].data_ptr() == y[j].data_ptr() and b[1].shape == y[j].shape for j, b in enumerate(batches)) else None
    return batches

  def close(self):
    _stop_producer(self)


class ShardStream(BatchStream):
  """`BatchStream` fed by the native streaming reader (`native/py_loader`): nothing but the pinned ring lives in host memory."""

  def __init__(self, paths, batch_size, device, seed=0, shuffle=True, depth=2, transform=None, readers=1, part=0, parts=1, pool=0, min_after_dequeue=-1,
               subset=None):
    """`subset`: the global record indices (shards in the order of `paths`, then records) this stream serves instead of `part`/`parts`."""
    from .. import native
    self._lib = native.library("py_loader")
    lib = self._lib
    lib.agb_loader_open.restype = ctypes.c_void_p
    lib.agb_loader_open_subset.restype = ctypes.c_void_p
    lib.agb_loader_last_error.restype = ctypes.c_char_p
    lib.agb_loader_next.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    lib.agb_loader_info.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    lib.agb_loader_close.argtypes = [ctypes.c_void_p]
    names = (ctypes.c_char_p * len(paths))(*[str(p).encode() for p in paths])
    common = (names, ctypes.c_int(len(paths)), ctypes.c_int(int(batch_size)), ctypes.c_int(max(1, int(readers))), ctypes.c_ulonglong(seed & (2 ** 64 - 1)),
              ctypes.c_int(1 if shuffle else 0), ctypes.c_longlong(pool), ctypes.c_longlong(min_after_dequeue))
    if subset is None:
      self._handle = lib.agb_loader_open(*common, ctypes.c_int(part), ctypes.c_int(parts))
    else:
      records = sum(read_shard_header(p)["count"] for p in paths)
      subset = np.asarray(subset, dtype=np.int64)
      if subset.size and (subset.min() < 0 or subset.max() >= records):
        raise tools.UserException("Shard subset indices must lie in [0, %d)" % records)
      member = np.zeros(-(-records // 64) * 64, dtype=bool)
      member[subset] = True
      bitmap = np.packbits(member.reshape(-1, 64)[:, ::-1], axis=1).view(">u8").astype(np.uint64).reshape(-1)
      self._handle = lib.agb_loader_open_subset(*common, bitmap.ctypes.data_as(ctypes.c_void_p), ctypes.c_ulonglong(records))
    if not self._handle:
      raise tools.UserException("Cannot open the dataset shards: " + lib.agb_loader_last_error().decode())
    info = (ctypes.c_ulonglong * 6)()
    lib.agb_loader_info(self._handle, info)
    self.total = int(info[0])
    self.batch = int(batch_size)
    self.device = _indexed(device)
    self.shuffle, self.transform = shuffle, transform
    self._cuda = self.device.type == "cuda"
    self._depth = depth
    self._queue, self._thread, self._stop, self._error = None, None, False, None
    self.sample_shape, self.sample_dtype = (int(info[2]), int(info[3]), int(info[4])), torch.uint8
    self.h2d_bytes = self.batch * int(info[5]) + self.batch * 8

  def _host_batch(self, slot=None):
    if slot is None:
      slot = (torch.empty((self.batch,) + self.sample_shape, dtype=torch.uint8), torch.empty(self.batch, dtype=torch.int64))
    if self._lib.agb_loader_next(self._handle, ctypes.c_void_p(slot[0].data_ptr()), ctypes.c_void_p(slot[1].data_ptr())) != 0:
      raise tools.UserException("Dataset reader failed: " + self._lib.agb_loader_last_error().decode())
    return slot

  def close(self):
    super().close()
    thread = self._thread
    if thread is not None and thread.is_alive():
      thread.join(timeout=2.0)
    if self._handle and (thread is None or not thread.is_alive()):
      self._lib.agb_loader_close(self._handle)
      self._handle = None

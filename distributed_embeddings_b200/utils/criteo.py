"""Criteo data sources for the DLRM example.

``RawBinaryDataset`` reads the *split binary* Criteo format (``label.bin`` bool, ``numerical.bin``
fp16, ``cat_<i>.bin`` int8/16/32 chosen by cardinality) with positional reads and a background
prefetch thread; batches land in pinned host memory so the H2D copy can be asynchronous.
``DummyDataset`` yields constant batches for benchmarking.

Capability parity: reference examples/dlrm/utils.py:116-307.
"""
from __future__ import annotations

import math
import os
import queue
import threading
from typing import Optional, Sequence

import numpy as np
import torch


def get_categorical_feature_type(size: int):
  for t in (np.int8, np.int16, np.int32):
    if size < np.iinfo(t).max:
      return t
  raise RuntimeError(f"Categorical feature of size {size} is too big for defined types")


class DummyDataset:
  """Constant synthetic batches (model-parallel categorical inputs unless ``dp_input``).
  ``hotness``: ids per sample of each of the ``num_tables`` features; given, every categorical
  tensor is ``[b, h_f]`` (multi-hot), else ``[b]``."""

  def __init__(self, batch_size: int, num_numerical: int, num_workers: int, num_tables: int,
               is_train: bool, dp_input: bool, num_batches: int,
               hotness: Optional[Sequence[int]] = None):
    lb = batch_size // num_workers
    self.numerical = torch.zeros(lb, num_numerical)
    cb = lb if dp_input else batch_size
    if hotness is None:
      self.categorical = [torch.zeros(cb, dtype=torch.int64) for _ in range(num_tables)]
    else:
      self.categorical = [torch.zeros(cb, int(h), dtype=torch.int64) for h in hotness]
    self.labels = torch.ones(lb if is_train else batch_size, 1)
    self.num_batches = num_batches

  def __len__(self):
    return self.num_batches

  def __getitem__(self, idx):
    if idx >= self.num_batches:
      raise IndexError
    return self.numerical, self.categorical, self.labels

  def __iter__(self):
    for i in range(self.num_batches):
      yield self[i]


class RawBinaryDataset:
  """Split-binary Criteo reader.

  Args:
    data_path: directory holding ``train/`` and ``test/`` sub-directories.
    batch_size: global batch size (one record of every file per sample).
    numerical_features: number of numerical features to load (0 = none).
    categorical_features: ids of the categorical features this rank needs.
    categorical_feature_sizes: cardinalities (select the on-disk integer type).
    prefetch_depth: batches read ahead by the background thread.
    offset / lbs: this rank's slice ``[offset, offset + lbs)`` of the global batch for the
      data-parallel tensors (numerical, labels, and categorical when ``dp_input``).
  """

  def __init__(self, data_path: str, batch_size: int = 1, numerical_features: int = 0,
               categorical_features: Optional[Sequence[int]] = None,
               categorical_feature_sizes: Optional[Sequence[int]] = None, prefetch_depth: int = 10,
               drop_last_batch: bool = False, valid: bool = False, offset: int = -1, lbs: int = -1,
               dp_input: bool = False, pin_memory: bool = True):
    data_path = os.path.join(data_path, "test" if valid else "train")
    self._bs = batch_size
    self._label_bytes = np.dtype(np.bool_).itemsize * batch_size
    self._num_feat = numerical_features
    self._num_bytes = numerical_features * np.dtype(np.float16).itemsize * batch_size
    self._cat_types = [get_categorical_feature_type(s) for s in (categorical_feature_sizes or [])]
    self._cat_bytes = [np.dtype(t).itemsize * batch_size for t in self._cat_types]
    self._cat_ids = list(categorical_features) if categorical_features else []
    rnd = math.floor if drop_last_batch else math.ceil
    self._label_file = os.open(os.path.join(data_path, "label.bin"), os.O_RDONLY)
    self._num_entries = int(rnd(os.fstat(self._label_file).st_size / self._label_bytes))
    self._num_file = None
    if numerical_features > 0:
      self._num_file = os.open(os.path.join(data_path, "numerical.bin"), os.O_RDONLY)
      n = rnd(os.fstat(self._num_file).st_size / self._num_bytes)
      if n != self._num_entries:
        raise ValueError(f"Size mismatch in data files. Expected: {self._num_entries}, got: {n}")
    self._cat_files = []
    for cid in self._cat_ids:
      f = os.open(os.path.join(data_path, f"cat_{cid}.bin"), os.O_RDONLY)
      n = rnd(os.fstat(f).st_size / self._cat_bytes[cid])
      if n != self._num_entries:
        raise ValueError(f"Size mismatch in data files. Expected: {self._num_entries}, got: {n}")
      self._cat_files.append(f)
    self._depth = min(prefetch_depth, self._num_entries)
    self.offset, self.lbs, self.valid, self.dp_input = offset, lbs, valid, dp_input
    self._pin = pin_memory and torch.cuda.is_available()

  def __len__(self):
    return self._num_entries

  def _pinned(self, arr: np.ndarray) -> torch.Tensor:
    if not arr.flags.writeable:  # np.frombuffer views of the bytes just read are read-only
      arr = arr.copy()
    t = torch.from_numpy(arr)
    return t.pin_memory() if self._pin else t

  def _get_item(self, idx: int):
    lab = np.frombuffer(os.pread(self._label_file, self._label_bytes, idx * self._label_bytes),
                        dtype=np.bool_).astype(np.float32).reshape(-1, 1)
    num = None
    if self._num_file is not None:
      raw = os.pread(self._num_file, self._num_bytes, idx * self._num_bytes)
      num = np.frombuffer(raw, dtype=np.float16).reshape(-1, self._num_feat)
    cats = []
    for cid, f in zip(self._cat_ids, self._cat_files):
      raw = os.pread(f, self._cat_bytes[cid], idx * self._cat_bytes[cid])
      cats.append(np.frombuffer(raw, dtype=self._cat_types[cid]).astype(np.int32))
    if self.offset >= 0:
      sl = slice(self.offset, self.offset + self.lbs)
      if not self.valid:
        lab = lab[sl]
      if num is not None:
        num = num[sl]
      if self.dp_input:
        cats = [c[sl] for c in cats]
    return (self._pinned(np.ascontiguousarray(num)) if num is not None else None,
            [self._pinned(np.ascontiguousarray(c)) for c in cats],
            self._pinned(np.ascontiguousarray(lab)))

  def __getitem__(self, idx: int):
    if idx >= self._num_entries:
      raise IndexError
    return self._get_item(idx)

  def __iter__(self):
    """Sequential iteration with a background prefetch thread."""
    q: "queue.Queue" = queue.Queue(maxsize=max(1, self._depth))
    stop = threading.Event()

    def producer():
      for i in range(self._num_entries):
        if stop.is_set():
          return
        q.put(self._get_item(i))
      q.put(None)

    t = threading.Thread(target=producer, daemon=True)
    t.start()
    try:
      while True:
        item = q.get()
        if item is None:
          return
        yield item
    finally:
      stop.set()

  def __del__(self):
    for f in [getattr(self, "_label_file", None), getattr(self, "_num_file", None)] + \
        list(getattr(self, "_cat_files", [])):
      if f is not None:
        try:
          os.close(f)
        except OSError:
          pass

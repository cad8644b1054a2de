"""Loader for the native sm_90a extension and numpy mirrors of its descriptor structs."""
from __future__ import annotations

import os
import threading

import numpy as np
import torch

_PKG_DIR = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO_PATH = os.path.join(_PKG_DIR, "_C.so")

_lock = threading.Lock()
_loaded = False
_error = None

# mirrors of de::InputDesc / de::TableDesc (ops/csrc/de_b200.h); sizes are checked at load time
INPUT_DESC = np.dtype([
    ("table", "<u8"),
    ("ids", "<u8"),
    ("offsets", "<u8"),
    ("ids_off", "<i8"),
    ("id_shift", "<i8"),
    ("sub_rows", "<i8"),
    ("row_base", "<i8"),
    ("width", "<i4"),
    ("hotness", "<i4"),
    ("dst_col", "<i4"),
    ("combiner", "<i4"),
    ("local_table", "<i4"),
    ("flags", "<i4"),
    ("item_off", "<i8"),
    ("pad1", "<i8"),
])
TABLE_DESC = np.dtype([
    ("weight", "<u8"),
    ("state0", "<u8"),
    ("state1", "<u8"),
    ("rows", "<i8"),
    ("key_base", "<i8"),
    ("width", "<i4"),
    ("pad", "<i4"),
])

# mirror of de::GradRoute: one contiguous piece of a requester-side gradient row -> its owner
GRAD_ROUTE = np.dtype([
    ("dst", "<u8"),
    ("dst_stride", "<i8"),
    ("src_col", "<i4"),
    ("width", "<i4"),
    ("dst_col", "<i4"),
    ("pad", "<i4"),
])
# mirror of de::CacheRemap: one cached input of the offload cache's id remap (offload_cache.cu)
CACHE_REMAP = np.dtype([
    ("ids", "<u8"),
    ("n", "<i8"),
    ("id_shift", "<i8"),
    ("sub_rows", "<i8"),
    ("row_base", "<i8"),
    ("out_off", "<i8"),
])
SYNC_STATE_WORDS = 64
DTYPE_CODE = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}

OPT_SGD, OPT_ADAGRAD, OPT_ROWWISE_ADAGRAD, OPT_ADAM, OPT_EMIT = 0, 1, 2, 3, 4
OPT_ROWWISE_ADAM = 5
OPT_FTRL = 6
OPT_MOMENTUM = 7
MAX_PEERS = 16


def load(required: bool = False) -> bool:
  """Load ``_C.so`` once.  Returns True when the native ops are available."""
  global _loaded, _error
  if _loaded:
    return True
  with _lock:
    if _loaded:
      return True
    if _error is not None and not required:
      return False
    try:
      if not os.path.exists(SO_PATH):
        raise FileNotFoundError(
            f"{SO_PATH} is missing - run `python -m distributed_embeddings_b200.ops._build` "
            "(or `make`) to compile the sm_90a kernels")
      torch.ops.load_library(SO_PATH)
      sizes = list(torch.ops.de_b200.struct_sizes())
      mine = [INPUT_DESC.itemsize, TABLE_DESC.itemsize, MAX_PEERS, GRAD_ROUTE.itemsize,
              SYNC_STATE_WORDS, CACHE_REMAP.itemsize]
      if sizes != mine:
        raise RuntimeError(f"descriptor layout mismatch: native {sizes} vs python {mine} "
                           "(stale _C.so? rebuild with python -m distributed_embeddings_b200.ops._build)")
      _loaded = True
      return True
    except Exception as e:  # pylint: disable=broad-except
      _error = e
      if required:
        raise
      return False


def available() -> bool:
  return load(required=False)


# number of kernels each native op launches (for the benchmark's launch accounting)
_KERNELS_PER_OP = {
    "lookup_fwd": 1, "scatter_add_bwd": 1, "sort_items": 12, "segment_update": 1,
    "sync_only": 1, "push_segments": 1, "push_grad": 1, "rowslice_reduce": 1,
    "embedding_lookup_fwd": 1, "embedding_scatter_add": 1, "embedding_lookup_grad": 14,
    "row_to_split": 1, "hash_init": 1, "integer_lookup": 1, "barrier": 1, "allreduce": 1,
    "gather_segments": 1, "gather_ragged": 1, "copy_cast_2d": 1, "dense_sgd": 1, "interact_fwd": 1, "interact_bwd": 1,
    "dense_adagrad": 1, "dense_adam": 1, "dense_momentum": 1, "cross_fwd": 1, "cross_bwd": 1, "cross_dx0": 1,
    "relu_bwd_bias": 1, "head_loss": 1, "head_eval": 1, "select_copy": 1, "cast_pad": 1, "gemm_tn_bias_act": 1, "gemm_dgrad_relu_bias": 1,
    "auc_append": 1, "radix_sort_keys32": 12, "auc_count": 3,
}
_launches = 0


class _OpsProxy:
  """Forwards to ``torch.ops.de_b200`` and counts kernel launches."""

  def __init__(self, ns):
    self._ns = ns
    self._cache = {}

  def __getattr__(self, name):
    fn = self._cache.get(name)
    if fn is None:
      raw = getattr(self._ns, name)
      k = _KERNELS_PER_OP.get(name, 0)

      def fn(*args, __raw=raw, __k=k, **kwargs):
        global _launches
        _launches += __k
        return __raw(*args, **kwargs)

      self._cache[name] = fn
    return fn


_proxy = None


def reset_launch_count():
  global _launches
  _launches = 0


def launch_count() -> int:
  return _launches


def require():
  """Fail loudly when a CUDA tensor reaches an op but the extension is missing."""
  global _proxy
  if not load(required=False):
    raise RuntimeError(
        "distributed_embeddings_b200: the native sm_90a extension is required for CUDA tensors "
        f"but could not be loaded ({_error!r}). There is no eager fallback on GPU.")
  if _proxy is None:
    _proxy = _OpsProxy(torch.ops.de_b200)
  return _proxy


def ops():
  return require()


def upload_struct_array(arr: np.ndarray, device) -> torch.Tensor:
  """Copy a numpy struct array to the device as raw bytes."""
  raw = torch.from_numpy(np.frombuffer(arr.tobytes(), dtype=np.uint8).copy())
  return raw.to(device)

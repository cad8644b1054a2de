"""The fused engine's CUDA kernels against the plan interpreter (parallel/dry_run.py), at world
sizes 2-8 on one GPU.

Every rank of a plan runs in one process (``dry_run.run_ranks``).  Each op call of every engine
is replayed: the interpreter's ``DryOps`` runs on host memory (the oracle; it bounds-checks every
access), then the real ``torch.ops.de_b200`` op runs with identical arguments on device mirrors of
every registered host buffer, and every mirror must equal its host buffer afterwards.  The
kernels only dereference the pointers they are given, so the "peer" buffers of the other ranks
can be separate allocations on the same device.

* Mirrors: one device buffer per registered host storage, same size, same offsets (host storages
  are >= 64-byte aligned, device ones >= 256-byte aligned, so every pointer keeps its alignment
  modulo 16 and the vec4 / vec8 / staged choices the engine made from host pointers stay valid),
  followed by a guard zone of a fixed byte pattern that must survive every op.
* Pointers inside descriptor blobs, pointer lists and scalar pointers are translated to the
  mirrors; a non-zero pointer outside every registered buffer raises before any launch.
* Every real op gets ``sync=[]``: the interpreter already did the host-side wait, and the
  signalling protocol needs real peers (``test_dist_gpu.py``).  ``stream_push`` polls progress
  counters without a timeout then, so the interpreter checks first that they are complete.
* Ranks run one at a time: a rank thread holds a token and yields it only while it waits in a
  barrier, so no rank's host-side writes (staging its ids) can race another rank's comparison.
* Data sit on a coarse dyadic grid with a power-of-two learning rate and power-of-two mean
  weights: every fp32 sum is exact in any order, so pooling, scatter-adds and SGD must match bit
  for bit.  Exceptions, stated where they apply: Adagrad / row-wise Adagrad / Adam (nvcc contracts
  to FMA: ``OPT_ULPS`` fp32 ulps, one ulp of a 16-bit table), and world size 3 (the gradient scale
  1/3 is not dyadic, so atomic SGD sums depend on their order: ``INEXACT_ULPS``).
* After every op the mirrors are reset from the host buffers, so a failure names the first op,
  rank, buffer and element that diverged.

Kernel-authoritative updates (``MirrorWorld(authoritative=True)``, ``test_update_conformance.py``):
the fp32 math of row-wise Adam and FTRL (``powf``, ``(P(n') - P(n)) / lr``, the ``l1``
threshold) may differ from the interpreter's torch ops by far more than a few ulps, so no ulp
tolerance can be both safe and tight.  There, a ``segment_update`` with an optimizer still runs
the interpreter first (the bounds-checked oracle for addressing), then the kernel, and:

* in the weight and state buffers of the op's tables, every row whose key is not among the op's
  ``n_unique`` sorted keys must be bit-identical to the host, and the touched rows are copied from
  the mirrors into the host buffers, so later ops, later steps and the test's float64 model all
  see the kernel's numbers;
* every other buffer is compared as above, the balanced route's ``scratch`` included (it must
  be all zero again after the op);
* zero weights are then stored as +0.0: the kernels keep the sign of a -0.0 weight through a
  one-id pool, the interpreter's sum does not.

With at most two ids per sample, every pooled sum has at most two terms and is exact in any
order, so the other ops stay bit-exact on the non-dyadic values the updates produce.

A CPU self-check runs the same harness with a second ``DryWorld`` as the "device" and the
interpreter as the "kernels": it must reproduce the interpreter byte for byte.
"""
import bisect
import collections
import functools
import inspect
import threading

import numpy as np
import pytest
import torch

from distributed_embeddings_b200.ops import _native
from distributed_embeddings_b200.ops._native import GRAD_ROUTE, INPUT_DESC, TABLE_DESC
from distributed_embeddings_b200.parallel import dry_run
from distributed_embeddings_b200.parallel.embedding_optimizers import BY_CODE
from test_dry_run import run_inplace_plan, run_plan  # pylint: disable=wrong-import-order

GUARD = 256          # guard bytes behind every mirror
GUARD_BYTE = 0xA5
OPT_ULPS = 4         # Adagrad / row-wise Adagrad / Adam, fp32 tables and state
INEXACT_ULPS = 16    # world size 3: order-dependent atomic sums of non-dyadic products
WEIGHT_FLOOR = 1.0   # ulps of weights are taken at >= this magnitude: updates of O(lr) cancel

# kinds of the op arguments that need translation (names as in DryOps)
_SPECS = {
    "lookup_fwd": {"descs": "desc", "src_ptrs": "ptrs", "dst_ptrs": "ptrs", "sync": "sync"},
    "scatter_add_bwd": {"descs": "desc", "src_ptrs": "ptrs", "grad_ptrs": "ptrs",
                        "scale_ptr": "ptr", "sync": "sync"},
    "push_segments": {"segs": "tensor", "src": "tensor", "dst_ptrs": "ptrs", "sync": "sync"},
    "push_grad": {"routes": "route", "src": "tensor", "sync": "sync"},
    "stream_push": {"src_ptrs": "ptrs", "dst_ptrs": "ptrs", "counters": "tensor", "sync": "sync"},
    "rowslice_reduce": {"partial": "tensor", "out_ptr": "ptr", "cols": "tensor"},
    "gather_segments": {"segs": "tensor", "src_ptrs": "ptrs", "dst": "tensor"},
    "gather_ragged": {"rsegs": "tensor", "val_ptrs": "ptrs", "split_ptrs": "ptrs",
                      "dst_vals": "tensor", "goff": "tensor"},
    "copy_cast_2d": {"src": "tensor", "dst_ptr": "ptr"},
    "sort_items": {"descs": "desc", "tables": "tdesc", "src_ptrs": "ptrs"},
    "segment_update": {"descs": "desc", "tables": "tdesc", "grad_ptrs": "ptrs", "keys": "tensor",
                       "items": "tensor", "seg": "tensor", "n_unique": "tensor", "lr_ptr": "ptr",
                       "emit_keys": "tensor", "emit_rows": "tensor", "scratch": "tensor",
                       "step_ptr": "ptr"},
}
_BLOBS = {"desc": (INPUT_DESC, ("table", "ids", "offsets")),
          "tdesc": (TABLE_DESC, ("weight", "state0", "state1")),
          "route": (GRAD_ROUTE, ("dst",))}

# replayed op calls per kernel path, over the whole module (printed at its end)
REPLAYED = collections.Counter()


class CudaDevice:
  """The real kernels, on the current GPU."""

  def __init__(self):
    assert _native.load(required=True)
    self.device = torch.device("cuda", torch.cuda.current_device())

  def alloc(self, nbytes):
    return torch.empty(nbytes, dtype=torch.uint8, device=self.device)

  def op(self, name, rank):  # pylint: disable=unused-argument
    return getattr(torch.ops.de_b200, name)

  def copy(self, t):
    return t.to(self.device)

  def synchronize(self):
    torch.cuda.synchronize(self.device)


class HostDevice:
  """CPU self-check: the mirrors are host buffers registered in a second ``DryWorld`` (the only
  buffers it knows, so an untranslated pointer is "outside any buffer"), and the "kernels" are
  the interpreter's ops on that world."""

  def __init__(self):
    self.world = dry_run.DryWorld(1)
    self.device = torch.device("cpu")

  def alloc(self, nbytes):
    t = torch.empty(nbytes, dtype=torch.uint8)
    self.world.register(t)
    return t

  def op(self, name, rank):
    return getattr(dry_run.DryOps(self.world, rank), name)

  def copy(self, t):
    return t.clone()

  def synchronize(self):
    pass


def _ordered16(raw: torch.Tensor) -> np.ndarray:
  """16-bit floats as integers that are consecutive for neighbouring values."""
  v = raw.view(torch.int16).numpy().astype(np.int64)
  return np.where(v < 0, -(v & 0x7FFF), v)


class MirrorWorld(dry_run.DryWorld):
  """A ``DryWorld`` whose engines replay every op on device mirrors (see the module doc)."""

  def __init__(self, world_size, device, inexact=False, authoritative=False):
    super().__init__(world_size)
    self.dev = device
    self.inexact = inexact
    self.authoritative = authoritative
    self.token = threading.Lock()
    self._holder = None
    self.mirrors = {}  # start of a registered host storage -> its mirror (+ padding + guard)
    self.all_ops = []

  # -- one rank at a time --------------------------------------------------------------------
  def make_ops(self, rank):
    ops = MirrorOps(self, rank)
    self.all_ops.append(ops)
    return ops

  def run_rank(self, fn, rank):
    with self.token:
      self._holder = threading.get_ident()
      try:
        return fn(rank)
      finally:
        self._holder = None

  def _yielding(self, wait):
    held = self._holder == threading.get_ident()
    if held:
      self._holder = None
      self.token.release()
    try:
      return wait()
    finally:
      if held:
        self.token.acquire()
        self._holder = threading.get_ident()

  def barrier(self):
    self._yielding(super().barrier)

  def bcast(self, buf, owner, rank):
    return self._yielding(lambda: super(MirrorWorld, self).bcast(buf, owner, rank))

  # -- mirrors -------------------------------------------------------------------------------
  def _storages(self):
    with self.lock:
      return sorted(self._ranges.items())

  def upload(self):
    """Every mirror := its host buffer (creates the mirrors of new buffers)."""
    for start, end in self._storages():
      n = end - start
      m = self.mirrors.get(start)
      if m is None:
        m = self.dev.alloc((n + 15) // 16 * 16 + GUARD)
        m[n:].fill_(GUARD_BYTE)
        self.mirrors[start] = m
      m[:n].copy_(self.tensor(start, torch.uint8, n))

  def _find(self, ptr):
    with self.lock:
      i = bisect.bisect_right(self._starts, ptr) - 1
      if i >= 0 and ptr <= self._ranges[self._starts[i]]:
        return self._starts[i]
    return None

  def translate(self, ptr, what):
    ptr = int(ptr)
    if ptr == 0:
      return 0
    start = self._find(ptr)
    if start is None:
      raise RuntimeError(f"{what}: pointer {ptr:#x} lies outside every registered buffer; it "
                         "would reach a kernel as a host address")
    return self.mirrors[start].data_ptr() + (ptr - start)

  def translate_blob(self, blob, kind, what):
    dt, fields = _BLOBS[kind]
    arr = np.frombuffer(blob.numpy().tobytes(), dtype=dt).copy()
    for f in fields:
      arr[f] = [self.translate(p, f"{what}[{i}].{f}") for i, p in enumerate(arr[f])]
    return self.dev.copy(torch.from_numpy(np.frombuffer(arr.tobytes(), dtype=np.uint8).copy()))

  def mirror_of(self, t):
    """The view of the mirror that aliases host tensor ``t`` (None: not a registered buffer)."""
    if t.device.type != "cpu" or not t.numel():
      return None
    start = self._find(t.data_ptr())
    if start is None:
      return None
    off = t.data_ptr() - start
    assert off % t.element_size() == 0
    return self.mirrors[start].view(t.dtype).as_strided(t.shape, t.stride(),
                                                       off // t.element_size())

  # -- diagnostics ---------------------------------------------------------------------------
  def describe(self, start):
    """(name, dtype) of the registered storage at ``start``: engine attribute or DryBuf name."""
    def walk(name, v):
      if isinstance(v, torch.Tensor):
        yield name, v
      elif isinstance(v, dry_run.DryBuf):
        yield f"{v.name} (engine.{name})", v.local
      elif isinstance(v, (list, tuple)):
        for k, x in enumerate(v):
          yield from walk(f"{name}[{k}]", x)
      elif isinstance(v, dict):
        for k, x in v.items():
          yield from walk(f"{name}[{k}]", x)

    for ops in self.all_ops:
      e = ops.engine
      if e is None:
        continue
      cands = [(f"model-parallel table {m} weight", layer.embeddings)
               for m, layer in enumerate(e.mp_layers)]
      cands += [(f"replicated table {m} weight", layer.embeddings)
                for m, layer in enumerate(e.de.dp_layers)]
      for name, v in vars(e).items():
        cands += list(walk(name, v))
      for name, t in cands:
        if t.numel() and t.untyped_storage().data_ptr() == start:
          return f"rank {ops.rank} {name}", t.dtype
    return f"buffer at {start:#x}", torch.uint8

  def compare(self, what, tol=None, skip=()):
    """Every mirror == its host buffer, every guard intact.  ``tol``: ulps allowed in float
    buffers (fp32; 16-bit buffers: one ulp of their format); ``skip``: starts of storages whose
    contents are not compared (their guards are)."""
    self.dev.synchronize()
    for start, end in self._storages():
      n = end - start
      got = self.mirrors[start].cpu()
      want = self.tensor(start, torch.uint8, n)
      name = None
      if not bool((got[n:] == GUARD_BYTE).all()):
        name, _ = self.describe(start)
        k = int(torch.nonzero(got[n:] != GUARD_BYTE)[0])
        raise AssertionError(f"{what}: store behind the end of {name} ({n} bytes): guard byte "
                             f"{k} is {int(got[n + k]):#x}")
      if start in skip or torch.equal(got[:n], want):
        continue
      name, dtype = self.describe(start)
      esz = torch.empty((), dtype=dtype).element_size()
      bad = torch.nonzero(got[:n] != want).view(-1)
      if tol is not None and dtype.is_floating_point and n % esz == 0:
        a, b = got[:n].view(dtype), want.clone().view(dtype)
        if esz == 2:
          ok = np.abs(_ordered16(a) - _ordered16(b)) <= 1
        else:
          a, b = a.numpy(), b.numpy()
          floor = WEIGHT_FLOOR if "weight" in name else 0.0
          mag = np.maximum(np.maximum(np.abs(a), np.abs(b)), floor)
          ok = (a == b) | (np.abs(a - b) <= tol * np.spacing(mag.astype(np.float32)))
        if ok.all():
          continue
        e = int(np.nonzero(~ok)[0][0])
        raise AssertionError(f"{what}: {name} element {e}: kernel {float(a[e])!r} vs interpreter "
                             f"{float(b[e])!r} (more than {tol} ulps apart)")
      i = int(bad[0])
      e = i // esz
      a = got[e * esz:(e + 1) * esz].view(dtype) if (e + 1) * esz <= n else got[i:i + 1]
      b = want[e * esz:(e + 1) * esz].clone().view(dtype) if (e + 1) * esz <= n else want[i:i + 1]
      raise AssertionError(f"{what}: {name} differs in {bad.numel()} bytes, first at byte {i} "
                           f"(element {e} as {dtype}): kernel {a.tolist()} vs interpreter "
                           f"{b.tolist()}")


def _native_dtype(code):
  return {0: "fp32", 1: "bf16", 2: "fp16"}[int(code)]


def _tag(name, a):
  """Kernel path of one op call (for the census)."""
  if name == "lookup_fwd":
    tags = ["lookup_fwd"]
    if -(-a["batch"] // a["dst_batch"]) > 1:
      tags.append("lookup_fwd, several destinations")
    d = np.frombuffer(a["descs"].numpy().tobytes(), dtype=INPUT_DESC)[:a["n_inputs"]]
    if (d["flags"] & 1).any():
      tags.append("lookup_fwd, row-slice stores")
    return tags
  if name == "scatter_add_bwd":
    return ["scatter_add_bwd, " + ("staged" if a["staged"] else "unstaged") +
            (", vec8" if a["vec8"] else "")]
  if name == "segment_update":
    if a["kind"] == _native.OPT_EMIT:
      return ["segment_update, emit"]
    if a["scratch"] is not None and a["vec4"] and a["max_width"] <= 128:
      route = "balanced"
    else:
      route = "per-row " + ("vec4" if a["vec4"] else "vec1")
    kind = BY_CODE[a["kind"]]
    half_state = bool(a["state_dtype"]) and kind.elementwise_state
    tdt = _native_dtype(a["table_dtype"])
    tags = ["segment_update, " + route.split(" ")[0], f"segment_update, {route}, {kind.name}",
            f"segment_update, {tdt} table, {'bf16' if half_state else 'fp32'} state"]
    if a["table_dtype"]:
      tags += ["segment_update, 16-bit table", f"segment_update, {tdt} table, {kind.name}"]
    if half_state:
      tags.append(f"segment_update, bf16 state, {kind.name}")
    return tags
  return [name]


class MirrorOps(dry_run.DryOps):
  """``DryOps`` that replays every call on the device mirrors and compares."""

  def _replay(self, name, args, kwargs):
    w = self.world
    bound = inspect.signature(getattr(dry_run.DryOps, name)).bind(self, *args, **kwargs)
    bound.apply_defaults()
    a = dict(bound.arguments)
    a.pop("self")
    if "sync" in a:
      self._wait(a["sync"])  # the interpreter's host-side wait; the replay never waits
      a["sync"] = []
    what = f"{name} on rank {self.rank}"
    self._sync_registry()
    w.upload()
    spec = _SPECS[name]
    dev_args, copies = [], []
    for k, v in a.items():  # translate everything before anything runs
      kind = spec.get(k)
      if kind in _BLOBS:
        v = w.translate_blob(v, kind, f"{what}: {k}")
      elif kind == "ptrs":
        v = [w.translate(p, f"{what}: {k}[{i}]") for i, p in enumerate(v)]
      elif kind == "ptr":
        v = w.translate(v, f"{what}: {k}")
      elif kind == "tensor" and v is not None:
        m = w.mirror_of(v)
        if m is None:
          m = w.dev.copy(v)
          copies.append((k, a[k], m))
        v = m
      elif isinstance(v, np.generic):
        v = v.item()
      dev_args.append(v)
    want = getattr(super(), name)(**a)  # the oracle, on host memory
    got = w.dev.op(name, self.rank)(*dev_args)
    tol = None
    if name == "segment_update" and a["kind"] in (_native.OPT_ADAGRAD,
                                                  _native.OPT_ROWWISE_ADAGRAD, _native.OPT_ADAM):
      tol = OPT_ULPS
    if w.inexact and name in ("scatter_add_bwd", "segment_update"):
      tol = INEXACT_ULPS
    skip = set()
    adopt = w.authoritative and name == "segment_update" and a["kind"] != _native.OPT_EMIT
    if adopt:
      skip = self._adopt_update(what, a)
    w.compare(what, tol, skip)
    for k, host, dev in copies:
      self._compare_copy(what, name, a, k, host, dev.cpu())
    if name == "sort_items":
      self._compare_sort(what, a, want, [t.cpu() for t in got])
    for t in _tag(name, a):
      REPLAYED[t] += 1
    return want

  def _adopt_update(self, what, a):
    """Kernel-authoritative ``segment_update`` (see the module doc): rows of the op's tables that
    no key touched must be bit-identical in every weight and state buffer; the touched rows are
    copied from the mirrors into the host buffers.  Returns the storages ``compare`` must skip:
    these buffers, checked here."""
    w = self.world
    w.dev.synchronize()
    T = np.frombuffer(a["tables"].numpy().tobytes(), dtype=TABLE_DESC)[:a["n_tables"]]
    nu = int(a["n_unique"][0])
    keys = a["keys"][a["seg"][:nu].long()].long().numpy()
    opt = BY_CODE[a["kind"]]
    half_state = bool(a["state_dtype"]) and opt.elementwise_state
    skip = set()
    # storage -> (offset, rows, row bytes, table, slot, key base) of every weight / state buffer
    regions = collections.defaultdict(list)
    for m, t in enumerate(T):
      rows, width, base = int(t["rows"]), int(t["width"]), int(t["key_base"])
      mine = keys[(keys >= base) & (keys < base + rows)] - base
      slots = [("weight", t["weight"], width * (2 if a["table_dtype"] else 4))]
      for k, s in enumerate(opt.slots):
        slots.append((f"state{k}", t[f"state{k}"], 4 if s.per_row else
                      width * (2 if half_state else 4)))
      for label, ptr, row_bytes in slots:
        start = w._find(int(ptr))
        assert start is not None, f"{what}: table {m} {label} is not a registered buffer"
        off = int(ptr) - start
        regions[start].append((off, rows, row_bytes, m, label, base))
        host = w.tensor(int(ptr), torch.uint8, rows * row_bytes).view(rows, row_bytes)
        dev = w.mirrors[start][off:off + rows * row_bytes].view(rows, row_bytes)
        idx = torch.as_tensor(mine, dtype=torch.long)
        host[idx] = dev[idx.to(dev.device)].cpu()
    for start, parts in regions.items():
      skip.add(start)
      n = w._ranges[start] - start
      got = w.mirrors[start][:n].cpu()
      want = w.tensor(start, torch.uint8, n)
      if torch.equal(got, want):
        continue
      i = int(torch.nonzero(got != want)[0])
      name, _ = w.describe(start)
      for off, rows, row_bytes, m, label, base in parts:
        if off <= i < off + rows * row_bytes:
          row = (i - off) // row_bytes
          raise AssertionError(f"{what}: {name}: row {row} of table {m} ({label}, key "
                               f"{base + row}) changed, but no key of the op touched it")
      raise AssertionError(f"{what}: {name} differs at byte {i}, outside every table's rows")
    # a -0.0 weight (a 16-bit rounding or FTRL's closed form) pools to -0.0 through one id in the
    # kernels but to +0.0 in the interpreter's sum: later ops see the zero weights as +0.0
    tdt = {0: torch.float32, 1: torch.bfloat16, 2: torch.float16}[int(a["table_dtype"])]
    for t in T:
      wt = w.tensor(int(t["weight"]), tdt, int(t["rows"]) * int(t["width"]))
      wt[wt == 0] = 0
    return skip

  @staticmethod
  def _compare_copy(what, name, a, k, host, got):
    if name == "segment_update" and k in ("emit_keys", "emit_rows"):
      nu = int(a["n_unique"][0])
      keys = a["emit_keys"][:nu]
      assert torch.equal(got[:nu], host[:nu]) if k == "emit_keys" else True, \
          f"{what}: emit_keys differ"
      if k == "emit_rows":
        T = np.frombuffer(a["tables"].numpy().tobytes(), dtype=TABLE_DESC)[:a["n_tables"]]
        bases = [int(x) for x in T["key_base"]]
        sentinel = bases[-1] + int(T[-1]["rows"])
        for u in range(nu):
          key = int(keys[u])
          if key >= sentinel:
            continue
          width = int(T[bisect.bisect_right(bases, key) - 1]["width"])
          assert torch.equal(got[u, :width], host[u, :width]), \
              f"{what}: emitted row {u} (key {key}): kernel {got[u, :width].tolist()} vs " \
              f"interpreter {host[u, :width].tolist()}"
      return
    assert torch.equal(got.view(torch.uint8) if got.dtype == torch.bool else got, host), \
        f"{what}: argument {k} differs after the op"

  @staticmethod
  def _compare_sort(what, a, want, got):
    ks, its, seg, nu = want
    gk, gi, gs, gn = got
    assert torch.equal(gn, nu), f"{what}: n_unique kernel {gn.tolist()} vs {nu.tolist()}"
    n = int(nu[0])
    for label, x, y in (("keys", gk, ks), ("seg_start", gs[:n + 1], seg[:n + 1])):
      if not torch.equal(x, y):
        i = int(torch.nonzero(x != y)[0])
        raise AssertionError(f"{what}: sorted {label} differ first at {i}: kernel {int(x[i])} "
                             f"vs interpreter {int(y[i])}")
    # both sides sort stably; unused slots of ragged inputs (sentinel keys) hold no item
    live = ks < a["total_rows"] if a["prefill_sentinel"] else torch.ones_like(ks, dtype=bool)
    if not torch.equal(gi[live], its[live]):
      i = int(torch.nonzero((gi != its) & live)[0])
      raise AssertionError(f"{what}: sorted items differ first at {i} (key {int(ks[i])}): "
                           f"kernel {int(gi[i])} vs interpreter {int(its[i])}")


def _replayed(name):
  def op(self, *args, **kwargs):
    return self._replay(name, args, kwargs)  # pylint: disable=protected-access
  op.__name__ = name
  return op


for _name in _SPECS:
  setattr(MirrorOps, _name, _replayed(_name))


@pytest.fixture(scope="module", autouse=True)
def _census():
  yield
  if REPLAYED:
    print("\nreplayed op calls per kernel path:")
    for k in sorted(REPLAYED):
      print(f"  {k}: {REPLAYED[k]}")


def _host_world():
  return functools.partial(MirrorWorld, device=HostDevice())


def _ok(outcomes, least):
  assert outcomes.count("ok") >= least, outcomes


# ---------------------------------------------------------------------------------- CPU self-check
DYADIC = {"dyadic": True}


@pytest.mark.parametrize("world", [1, 2, 3, 4])
@pytest.mark.parametrize("kind", ["sgd", "adagrad", "none"])
def test_harness_reproduces_the_interpreter(world, kind):
  """With the interpreter as the "kernels", every replayed op must match byte for byte."""
  before = REPLAYED.copy()
  _ok([run_plan(21000 * world + s + len(kind), world, kind, profile=DYADIC,
                world_cls=_host_world()) for s in range(2)], 1)
  assert REPLAYED["lookup_fwd"] > before["lookup_fwd"]


@pytest.mark.parametrize("world", [2, 4])
def test_harness_reproduces_the_interpreter_ragged_and_streamed(world):
  _ok([run_plan(23000 * world + s, world, "adagrad", ragged=True, profile=DYADIC,
                world_cls=_host_world()) for s in range(2)], 1)
  _ok([run_inplace_plan(24000 * world + s, world, True, profile=DYADIC,
                        world_cls=_host_world()) for s in range(2)], 1)


def test_pointer_outside_every_buffer_is_refused_before_launch():
  """A descriptor pointer that no registered buffer contains must stop the replay before the
  op runs (on a GPU it would be a host address in a kernel)."""
  embs = [{"input_dim": 10, "output_dim": 8, "combiner": "sum"} for _ in range(2)]
  sim, des = dry_run.build_engines(embs, 1, _host_world())
  de = des[0]
  ids = [torch.randint(0, 10, (4, 2)) for _ in range(2)]
  dry_run.run_ranks(sim, lambda r: de(ids, concat=True))
  eng = de._engine
  calls = dict(eng.ops.calls)
  eng.cdesc_np[0]["ids"] = 64  # no buffer there
  eng._upload()
  with pytest.raises(RuntimeError, match="outside every registered buffer"):
    dry_run.run_ranks(sim, lambda r: eng._run_forward())
  assert eng.ops.calls.get("lookup_fwd") == calls.get("lookup_fwd"), "the op ran"


def test_guard_zone_and_mismatch_are_reported():
  """A store behind a buffer's end and a wrong value are both named (buffer, element)."""
  world = MirrorWorld(1, HostDevice())
  t = torch.zeros(10, dtype=torch.float32)
  world.register(t)
  world.upload()
  start = t.untyped_storage().data_ptr()
  world.compare("no-op")
  world.mirrors[start][40] = 0
  with pytest.raises(AssertionError, match="guard byte 0"):
    world.compare("overrun")
  world.mirrors[start][40:] = GUARD_BYTE
  world.compare("restored")
  world.mirrors[start][:40].view(torch.float32)[3] = 1.0
  with pytest.raises(AssertionError, match="first at byte 14"):
    world.compare("value")


# ------------------------------------------------------------------------------------------ GPU
_DEVICE = []


def _gpu_world(inexact=False, made=None):
  if not _DEVICE:
    _DEVICE.append(CudaDevice())

  def make(n):
    w = MirrorWorld(n, _DEVICE[0], inexact=inexact or n == 3)
    if made is not None:
      made.append(w)
    return w
  return make


def _delta(before):
  return {k: v - before.get(k, 0) for k, v in REPLAYED.items() if v - before.get(k, 0)}


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("kind", ["sgd", "adagrad", "rowwise_adagrad", "adam", "none"])
def test_gpu_random_plans(world, kind):
  n = 3 if world < 8 else 2
  before = REPLAYED.copy()
  _ok([run_plan(31000 * world + 7 * s + len(kind), world, kind, profile=DYADIC,
                world_cls=_gpu_world()) for s in range(n)], 1)
  if kind != "none":  # weight decay (dyadic: exact on the grid) at grad_scale = 1 / world
    _ok([run_plan(32000 * world + 7 * s + len(kind), world, kind, profile=DYADIC,
                  world_cls=_gpu_world(), weight_decay=0.25) for s in range(2)], 1)
  d = _delta(before)
  assert d.get("lookup_fwd, several destinations", 0) > 0, d
  if kind == "none":
    assert d.get("segment_update, emit", 0) > 0, d


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3, 4])
@pytest.mark.parametrize("kind", ["sgd", "adagrad"])
def test_gpu_random_plans_ragged(world, kind):
  before = REPLAYED.copy()
  _ok([run_plan(33000 * world + s, world, kind, ragged=True, profile=DYADIC,
                world_cls=_gpu_world()) for s in range(3)], 1)
  d = _delta(before)
  assert d.get("gather_ragged", 0) > 0 and d.get("gather_segments", 0) >= 0, d


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 4])
def test_gpu_random_plans_bf16_activations(world):
  _ok([run_plan(35000 * world + s, world, "sgd", torch.bfloat16, profile=DYADIC,
                world_cls=_gpu_world()) for s in range(3)], 1)


@pytest.mark.gpu
@pytest.mark.parametrize("table_dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("kind", ["sgd", "adam", "none"])
def test_gpu_random_plans_half_tables(world, kind, table_dtype):
  before = REPLAYED.copy()
  _ok([run_plan(37000 * world + s + len(kind), world, kind,
                profile=dict(DYADIC, table_dtype=table_dtype), world_cls=_gpu_world())
       for s in range(2)], 1)
  if kind != "none":
    assert _delta(before).get("segment_update, 16-bit table", 0) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3, 4, 8])
@pytest.mark.parametrize("streamed", [False, True])
def test_gpu_backward_inplace_plans(world, streamed):
  """The hand-scheduled steps' backward: ``push_grad`` through ``routes_all``, or through
  ``routes_stage`` followed by the ``stream_push`` copy kernel."""
  before = REPLAYED.copy()
  _ok([run_inplace_plan(39000 * world + 17 * s + int(streamed), world, streamed, profile=DYADIC,
                        world_cls=_gpu_world()) for s in range(5)], 1)
  d = _delta(before)
  assert d.get("push_grad", 0) > 0, d
  if streamed:
    assert d.get("stream_push", 0) > 0, d


# widths 1-3 take the scalar path; 64 fp32 / 128 bf16 columns are the staged scatter's limit;
# above 128 rows take several column passes and the update switches to the per-row kernel
SCALE = {"dyadic": True, "rows": (200, 2000), "widths": (1, 2, 3, 12, 36, 64, 128, 136, 192, 256),
         "hotness": (1, 1, 2, 5, 9, 16, 40), "local_batch": tuple(range(33, 101)),
         "ragged_len": 24, "power_law": True, "out_of_table": True}


@pytest.mark.gpu
@pytest.mark.parametrize("world,kind,seed", [(2, "sgd", 0), (2, "adagrad", 1), (3, "adam", 2),
                                             (4, "none", 3), (4, "adam", 4),
                                             (8, "sgd", 5), (2, "sgd", 6), (4, "adagrad", 7)])
def test_gpu_scale_profile(world, kind, seed):
  """Several 32-sample tiles per destination with a partial last one, rows wider than one pass,
  the 8-way multi-hot unroll, power-law ids (hot rows spanning many 32-item chunks of the
  balanced update), row-sliced tables fed ids outside the table, mixed widths per launch."""
  before = REPLAYED.copy()
  _ok([run_plan(41000 + 100 * seed + s, world, kind, profile=SCALE, world_cls=_gpu_world())
       for s in range(2)], 1)
  assert _delta(before).get("lookup_fwd, several destinations", 0) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("table_dtype", [torch.bfloat16, torch.float16])
def test_gpu_scale_profile_half_tables(table_dtype):
  before = REPLAYED.copy()
  _ok([run_plan(43000 + s, 4, "adagrad", profile=dict(SCALE, table_dtype=table_dtype),
                world_cls=_gpu_world()) for s in range(2)], 1)
  assert _delta(before).get("segment_update, 16-bit table", 0) > 0


@pytest.mark.gpu
def test_gpu_scale_profile_ragged():
  _ok([run_plan(45000 + s, 2, "sgd", ragged=True, profile=SCALE, world_cls=_gpu_world())
       for s in range(2)], 1)


@pytest.mark.gpu
@pytest.mark.parametrize("staged,vec8", [("1", "0"), ("0", "0"), ("1", "1"), ("0", "1")])
def test_gpu_scatter_variants(monkeypatch, staged, vec8):
  """``DE_B200_SCATTER_STAGED`` (cp.async staged SGD scatter with in-warp dedup of duplicate
  ids, or plain atomics) and ``DE_B200_VEC8_GRAD`` (16-byte gradient loads), read when the
  engine lays out a batch shape; power-law ids give the staged path many duplicates."""
  monkeypatch.setenv("DE_B200_SCATTER_STAGED", staged)
  monkeypatch.setenv("DE_B200_VEC8_GRAD", vec8)
  prof = {"dyadic": True, "rows": (50, 400), "widths": (8, 16, 32, 64), "hotness": (1, 2, 4, 9),
          "local_batch": (40, 70), "power_law": True}
  made, before = [], REPLAYED.copy()
  outcomes = [run_plan(47000 + s, 2, "sgd", profile=prof, world_cls=_gpu_world(made=made))
              for s in range(4)]
  _ok(outcomes, 1)
  engines = [ops.engine for w in made for ops in w.all_ops if ops.engine is not None]
  if staged == "1":
    assert any(e.staged_update for e in engines)
  else:
    assert not any(e.staged_update for e in engines)
  assert any(e.vec8 for e in engines) == (vec8 == "1")
  d = _delta(before)
  want = "scatter_add_bwd, " + ("staged" if staged == "1" else "unstaged") + \
      (", vec8" if vec8 == "1" else "")
  assert d.get(want, 0) > 0, d

"""Plan interpreter: run the fused engine of *every rank of a plan* in one process, on the CPU.

The fused back end turns a sharding plan into device descriptors (``InputDesc`` / ``TableDesc``
arrays full of raw pointers and offsets, segment lists for the index exchange, column offsets into
peer output / gradient buffers).  That host-side logic is the part of the engine that depends on
the plan, and it is exactly what cannot be exercised without as many GPUs as ranks.  This module
executes it anyway:

* :class:`DryWorld` plays the machine: one host buffer per (rank, symmetric allocation), peer
  pointers are the real addresses of those buffers, flag barriers are ``threading.Barrier``;
* :class:`DryOps` implements the kernels' *addressing contract* in plain PyTorch - the same
  arguments as the CUDA ops (descriptor blobs, pointer lists, strides), every access bounds-checked
  against the registered buffers - so a wrong offset in a descriptor becomes a wrong number or an
  "address outside any buffer" error instead of a silent corruption on eight GPUs;
* every rank runs its unmodified :class:`FusedEngine` in its own thread.

Used by ``tests/test_dry_run.py`` to fuzz plans at world sizes 1-8 (forward, SGD / Adagrad /
row-wise Adagrad / Adam updates, sparse-gradient emission, ragged index exchange) and usable as a
pre-flight check of a scaled-down production plan (``build_engines`` + ``run_ranks``).  The
semantics mirrored here are documented at the
kernels: lookup_kernels.cu (lookup_fwd / scatter_add_bwd), sparse_update_kernels.cu (build_keys,
segment_update, apply_update), comm_kernels.cu (gather_segments, copy_cast_2d).
"""
from __future__ import annotations

import bisect
import ctypes
import threading
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from ..ops._native import GRAD_ROUTE, INPUT_DESC, MAX_PEERS, TABLE_DESC
from ..ops.stochastic_rounding import stochastic_round
from . import fused as _fused


class DryWorld:
  """Shared state of one simulated job."""

  def __init__(self, world_size: int):
    self.world_size = int(world_size)
    self.lock = threading.Lock()
    self._barrier = threading.Barrier(self.world_size)
    self._bufs: Dict[Tuple[int, int], torch.Tensor] = {}
    self._ranges: Dict[int, int] = {}  # start address -> end address of every registered buffer
    self._starts: List[int] = []       # sorted keys of _ranges
    self._keep: List[torch.Tensor] = []
    self.errors: List[BaseException] = []

  # -- symmetric buffers ---------------------------------------------------------------------
  def buffer(self, rank: int, index: int, nbytes: int) -> torch.Tensor:
    """The ``index``-th symmetric allocation of ``rank`` (created on first use by any rank)."""
    with self.lock:
      key = (rank, index)
      if key not in self._bufs:
        t = torch.zeros(max(int(nbytes), 16), dtype=torch.uint8)
        self._bufs[key] = t
        self._register_locked(t)
      t = self._bufs[key]
      if t.numel() < nbytes:
        raise RuntimeError(f"symmetric allocation {index} differs in size across ranks "
                           f"({t.numel()} vs {nbytes} bytes)")
      return t

  # -- address space -------------------------------------------------------------------------
  def _register_locked(self, t: torch.Tensor):
    st = t.untyped_storage()
    start = st.data_ptr()
    if start and start not in self._ranges:
      self._ranges[start] = start + st.nbytes()
      bisect.insort(self._starts, start)
      self._keep.append(t)

  def register(self, t: Optional[torch.Tensor]):
    if isinstance(t, torch.Tensor) and t.device.type == "cpu" and t.numel():
      with self.lock:
        self._register_locked(t)

  def check(self, ptr: int, nbytes: int, what: str = ""):
    if nbytes <= 0:
      return
    with self.lock:
      i = bisect.bisect_right(self._starts, ptr) - 1
      if i >= 0 and ptr + nbytes <= self._ranges[self._starts[i]]:
        return
    raise RuntimeError(f"address outside any buffer: {what} [{ptr:#x}, +{nbytes})")

  def tensor(self, ptr: int, dtype: torch.dtype, count: int, what: str = "") -> torch.Tensor:
    """Flat tensor aliasing ``count`` elements at ``ptr`` (bounds-checked)."""
    count = int(count)
    if count <= 0:
      return torch.empty(0, dtype=dtype)
    nbytes = count * torch.empty((), dtype=dtype).element_size()
    self.check(int(ptr), nbytes, what)
    raw = (ctypes.c_char * nbytes).from_address(int(ptr))
    return torch.frombuffer(raw, dtype=dtype, count=count)

  def make_ops(self, rank: int) -> "DryOps":
    """The ops object every engine of ``rank`` calls (a subclass may replay them elsewhere)."""
    return DryOps(self, rank)

  def run_rank(self, fn, rank: int):
    """Body of the thread of ``rank`` (see :func:`run_ranks`)."""
    return fn(rank)

  def barrier(self):
    self._barrier.wait(timeout=120)

  def bcast(self, buf: torch.Tensor, owner: int, rank: int) -> torch.Tensor:
    """Broadcast between the simulated ranks (threads): the cold-path collective behind
    ``get_weights`` / ``get_optimizer_state``."""
    if rank == owner:
      self._bcast_slot = buf.clone()
    self._barrier.wait(timeout=120)
    out = self._bcast_slot.clone()
    self._barrier.wait(timeout=120)
    return out


class DryBuf:
  """Stand-in for :class:`comm.SymmetricBuffer`."""

  def __init__(self, ctx: "DryCtx", index: int, nbytes: int, name: str):
    self.ctx, self.index, self.name = ctx, index, name
    self.nbytes = int(nbytes)
    self.local = ctx.world.buffer(ctx.rank, index, nbytes)

  def view(self, dtype: torch.dtype, shape, byte_offset: int = 0) -> torch.Tensor:
    n = 1
    for s in shape:
      n *= int(s)
    nbytes = n * torch.empty((), dtype=dtype).element_size()
    assert byte_offset + nbytes <= self.local.numel(), (self.name, byte_offset, nbytes)
    return self.local[byte_offset:byte_offset + nbytes].view(dtype).view(*shape)

  def peer_ptrs(self, byte_offset: int = 0) -> List[int]:
    w = self.ctx.world
    return [w.buffer(r, self.index, self.nbytes).data_ptr() + byte_offset
            for r in range(w.world_size)]


class DryCtx:
  """Stand-in for :class:`comm.CommContext`."""

  def __init__(self, world: DryWorld, rank: int):
    self.world, self.rank, self.world_size = world, rank, world.world_size
    self.device = torch.device("cpu")
    self.p2p = True
    self.group = None
    self._n_alloc = 0

  def alloc(self, nbytes: int, name: str = "") -> DryBuf:
    buf = DryBuf(self, self._n_alloc, nbytes, name)
    self._n_alloc += 1
    return buf

  def alloc_multicast(self, nbytes: int, name: str = ""):
    return None

  def barrier(self, channel: int = 0):
    if self.world_size > 1:
      self.world.barrier()

  def sync(self, wait: int = -1, wait_abs: int = -1, signal: int = -1, slot=None):
    """Signalling spec of the interpreter: an op that *waits* rendezvouses with all ranks first.
    Every rank issues the same op sequence and its own signalling op precedes its waiting op in
    program order, so a barrier at each wait gives exactly the ordering the flag words give."""
    if self.world_size == 1:
      return []
    return [-1, int(wait), int(wait_abs), int(signal), 0]

  def check_errors(self):
    pass


_IDT = {True: torch.int64, False: torch.int32}


class DryOps:
  """The CUDA ops' calling convention, executed with PyTorch on host memory."""

  def __init__(self, world: DryWorld, rank: int):
    self.world, self.rank = world, rank
    self.engine = None
    self.calls: Dict[str, int] = {}

  # -- helpers -------------------------------------------------------------------------------
  def _sync_registry(self):
    """Everything the engine owns is addressable (tables, id buffers, optimizer state, ...)."""
    e, w = self.engine, self.world
    if e is None:
      return
    for v in vars(e).values():
      if isinstance(v, torch.Tensor):
        w.register(v)
      elif isinstance(v, (list, tuple)):
        for x in v:
          w.register(x if isinstance(x, torch.Tensor) else None)
      elif isinstance(v, dict):
        for x in v.values():
          if isinstance(x, torch.Tensor):
            w.register(x)
          elif isinstance(x, (list, tuple)):
            for y in x:
              w.register(y if isinstance(y, torch.Tensor) else None)
    de = e.de
    for layer in list(de.dp_layers) + list(de.local_embedding_layers) + list(de.row_layers):
      for p in layer.parameters():
        w.register(p.data)

  def _count(self, name):
    self.calls[name] = self.calls.get(name, 0) + 1
    self._sync_registry()

  def _wait(self, sync):
    """Head wait of a kernel (see DryCtx.sync)."""
    if sync and (sync[1] >= 0 or sync[2] >= 0):
      self.world.barrier()

  _ADT = {0: torch.float32, 1: torch.bfloat16, 2: torch.float16}

  def sync_only(self, sync):
    self._count("sync_only")
    self._wait(sync)

  @staticmethod
  def _descs(blob: torch.Tensor, n: int, dtype=INPUT_DESC) -> np.ndarray:
    return np.frombuffer(blob.numpy().tobytes(), dtype=dtype)[:int(n)]

  def _ids_of(self, d, g0: int, g1: int, ids64: bool, src_ptrs, src_batch: int):
    """(values [n_total], lengths [g1-g0]) of samples g0..g1 of one input."""
    idt = _IDT[bool(ids64)]
    hot = int(d["hotness"])
    if int(d["offsets"]):
      offs = self.world.tensor(int(d["offsets"]) + g0 * 8, torch.int64, g1 - g0 + 1, "csr offsets")
      a, b = int(offs[0]), int(offs[-1])
      esz = 8 if ids64 else 4
      vals = self.world.tensor(int(d["ids"]) + a * esz, idt, b - a, "ragged ids")
      return vals.to(torch.int64), (offs[1:] - offs[:-1])
    esz = 8 if ids64 else 4
    if int(d["ids"]):
      vals = self.world.tensor(int(d["ids"]) + g0 * hot * esz, idt, (g1 - g0) * hot, "ids")
      return vals.to(torch.int64), torch.full((g1 - g0,), hot, dtype=torch.int64)
    # staged in the sources' buffers: sample g lives on rank g // src_batch
    parts = []
    for g in range(g0, g1):
      s, i = divmod(g, src_batch)
      parts.append(self.world.tensor(int(src_ptrs[s]) + (int(d["ids_off"]) + i * hot) * esz, idt,
                                     hot, "peer ids"))
    return torch.cat(parts).to(torch.int64), torch.full((g1 - g0,), hot, dtype=torch.int64)

  def _table(self, d, table_dtype: int = 0) -> torch.Tensor:
    """The rows a descriptor may address, in the launch's table dtype (bounds-checked at its
    element size)."""
    w = int(d["width"])
    rows = int(d["row_base"]) + int(d["sub_rows"])
    return self.world.tensor(int(d["table"]), self._ADT[int(table_dtype)], rows * w,
                             "table").view(rows, w)

  @staticmethod
  def _pool_index(lens: torch.Tensor) -> torch.Tensor:
    return torch.repeat_interleave(torch.arange(lens.numel()), lens)

  # -- forward -------------------------------------------------------------------------------
  def lookup_fwd(self, descs, n_inputs, batch, src_batch, dst_batch, dst_stride, src_ptrs,
                 dst_ptrs, rot, ids64, act_dtype, vec4, sync, tile_samples=32, table_dtype=0,
                 vec8=False):
    self._count("lookup_fwd")
    assert 1 <= tile_samples <= 32
    assert not vec8 or (vec4 and int(table_dtype) != 0), "vec8 is for 16-bit tables with vec4"
    self._wait(sync)
    odt = self._ADT[int(act_dtype)]
    osz = 4 if int(act_dtype) == 0 else 2
    for d in self._descs(descs, n_inputs):
      width, col = int(d["width"]), int(d["dst_col"])
      if vec4:
        assert width % 4 == 0 and col % 4 == 0 and dst_stride % 4 == 0, "vec4 alignment"
      if vec8:
        assert width % 8 == 0 and col % 8 == 0 and dst_stride % 8 == 0, "vec8 alignment"
        assert int(d["table"]) % 16 == 0, "vec8: 16-byte aligned table"
      table = self._table(d, table_dtype).float()  # rows are pooled in fp32
      for dd in range(-(-batch // dst_batch)):
        g0, g1 = dd * dst_batch, min(batch, (dd + 1) * dst_batch)
        ns = g1 - g0
        vals, lens = self._ids_of(d, g0, g1, ids64, src_ptrs, src_batch)
        ids = vals + int(d["id_shift"])
        ok = (ids >= 0) & (ids < int(d["sub_rows"]))
        rows = table[(int(d["row_base"]) + ids.clamp(0, max(int(d["sub_rows"]) - 1, 0)))]
        rows = rows * ok.unsqueeze(1).to(rows.dtype)
        seg = self._pool_index(lens)
        pooled = torch.zeros(ns, width).index_add_(0, seg, rows)
        hits = torch.zeros(ns, dtype=torch.int64).index_add_(0, seg, ok.to(torch.int64))
        if int(d["combiner"]) == 1:  # the kernels multiply by the fp32 reciprocal of n
          pooled = pooled * (1.0 / lens.clamp(min=1).to(pooled.dtype)).unsqueeze(1)
        # the destination row block of requester dd: rows [0, ns) x columns [col, col + width)
        last = (ns - 1) * dst_stride + col + width
        out = self.world.tensor(int(dst_ptrs[dd]), odt, last, "lookup destination")
        self.world.check(int(dst_ptrs[dd]), last * osz, "lookup destination")
        view = torch.as_strided(out, (ns, width), (dst_stride, 1), col)
        if int(d["flags"]) & 1:  # row slices: only samples with an id inside the shard store
          keep = hits > 0
          if int(d["flags"]) & 6:  # ... plus ids outside the whole table (zero rows), one-hot
            assert int(d["hotness"]) == 1
            low = (ids < 0) if int(d["flags"]) & 2 else torch.zeros_like(ok)
            high = (ids >= int(d["sub_rows"])) if int(d["flags"]) & 4 else torch.zeros_like(ok)
            keep = keep | low | high
          view[keep] = pooled[keep].to(odt)
        else:
          view.copy_(pooled.to(odt))

  # -- index exchange ------------------------------------------------------------------------
  def push_segments(self, segs, src, dst_ptrs, max_seg, sync):
    """Index push: segment {dst rank, src offset, dst offset, n} of the local staging buffer is
    stored into the id buffer of its owner."""
    self._count("push_segments")
    self._wait(sync)
    esz = src.element_size()
    flat = src.view(-1)
    for r, so, do, n in segs.tolist():
      assert n <= max_seg
      dst = self.world.tensor(int(dst_ptrs[r]) + do * esz, src.dtype, n, "id push destination")
      dst.copy_(flat[so:so + n])

  def push_grad(self, routes, n_routes, src, dst_dtype, scale, sync):
    """Gradient push: every route piece of the local gradient rows goes to its owner."""
    self._count("push_grad")
    self._wait(sync)
    R = np.frombuffer(routes.numpy().tobytes(), dtype=GRAD_ROUTE)[:int(n_routes)]
    ddt = self._ADT[int(dst_dtype)]
    dsz = 4 if int(dst_dtype) == 0 else 2
    rows = src.shape[0]
    covered = torch.zeros(src.shape[1], dtype=torch.int32)
    for r in R:
      w, sc, dc, stride = int(r["width"]), int(r["src_col"]), int(r["dst_col"]), int(r["dst_stride"])
      assert sc + w <= src.shape[1], "route piece outside the gradient row"
      covered[sc:sc + w] += 1
      last = (rows - 1) * stride + dc + w
      self.world.check(int(r["dst"]), last * dsz, "gradient push destination")
      out = self.world.tensor(int(r["dst"]), ddt, last, "gradient push destination")
      torch.as_strided(out, (rows, w), (stride, 1), dc).copy_(
          (src[:, sc:sc + w].float() * scale).to(ddt))

  def stream_push(self, src_ptrs, dst_ptrs, row_bytes, counters, chunk_rows, rows, blocks, sync):
    """Copy kernel of the streamed gradient push: the locally staged rows of every remote owner
    are forwarded to that owner's receive buffer.  The real kernel polls the producer's per-chunk
    row counters; here the producer has already run, so they must be complete."""
    self._count("stream_push")
    assert len(src_ptrs) == len(dst_ptrs) == len(row_bytes) and 0 < blocks
    n_chunks = -(-int(rows) // int(chunk_rows))
    assert counters.numel() >= n_chunks, "one progress counter per chunk"
    for c in range(n_chunks):
      want = min(int(chunk_rows), int(rows) - c * int(chunk_rows))
      assert int(counters[c]) == want, f"chunk {c}: {int(counters[c])} of {want} rows produced"
    for sp, dp, rb in zip(src_ptrs, dst_ptrs, row_bytes):
      assert rb % 16 == 0 and int(sp) % 16 == 0 and int(dp) % 16 == 0, "16-byte copies"
      n = int(rows) * int(rb)
      src = self.world.tensor(int(sp), torch.uint8, n, "streamed push staging")
      dst = self.world.tensor(int(dp), torch.uint8, n, "streamed push destination")
      dst.copy_(src)

  def rowslice_reduce(self, partial, out_ptr, out_stride, out_dtype, cols):
    self._count("rowslice_reduce")
    odt = self._ADT[int(out_dtype)]
    world, rows, _ = partial.shape
    red = partial.sum(dim=0)
    for sc, dc, w in cols.tolist():
      last = (rows - 1) * out_stride + dc + w
      out = self.world.tensor(int(out_ptr), odt, last, "row-slice destination")
      torch.as_strided(out, (rows, w), (out_stride, 1), dc).copy_(red[:, sc:sc + w].to(odt))

  def gather_segments(self, segs, src_ptrs, dst, max_seg):
    self._count("gather_segments")
    esz = dst.element_size()
    flat = dst.view(-1)
    for s, so, do, n in segs.tolist():
      assert n <= max_seg
      src = self.world.tensor(int(src_ptrs[s]) + so * esz, dst.dtype, n, "segment source")
      flat[do:do + n] = src

  def gather_ragged(self, rsegs, val_ptrs, split_ptrs, dst_vals, goff, b, max_cap):
    """Ragged index exchange: per local ragged input, concatenate every source rank's values in
    rank order and build the global-batch CSR offsets."""
    self._count("gather_ragged")
    esz = dst_vals.element_size()
    world = len(val_ptrs)
    flat = dst_vals.view(-1)
    for in_off, item_off, sp_off, g_off in rsegs.tolist():
      pos = 0
      goff[g_off] = 0
      for s in range(world):
        sp = self.world.tensor(int(split_ptrs[s]) + sp_off * 8, torch.int64, b + 1, "row splits")
        n = int(sp[-1])
        assert n <= max_cap, "ragged capacity exceeded"
        vals = self.world.tensor(int(val_ptrs[s]) + in_off * esz, dst_vals.dtype, n, "ragged src")
        flat[item_off + pos:item_off + pos + n] = vals
        goff[g_off + s * b + 1:g_off + (s + 1) * b + 1] = sp[1:] + pos
        pos += n

  def copy_cast_2d(self, src, dst_ptr, dst_stride, dst_dtype, scale):
    self._count("copy_cast_2d")
    rows, cols = src.shape
    ddt = self._ADT[int(dst_dtype)]
    out = self.world.tensor(int(dst_ptr), ddt, (rows - 1) * dst_stride + cols, "grad buffer")
    torch.as_strided(out, (rows, cols), (dst_stride, 1)).copy_((src.float() * scale).to(ddt))

  # -- backward ------------------------------------------------------------------------------
  def _grad_rows(self, d, dd, ns, grad_ptrs, grad_stride, act_dtype) -> torch.Tensor:
    gdt = self._ADT[int(act_dtype)]
    width, col = int(d["width"]), int(d["dst_col"])
    last = (ns - 1) * grad_stride + col + width
    g = self.world.tensor(int(grad_ptrs[dd]), gdt, last, "gradient source")
    return torch.as_strided(g, (ns, width), (grad_stride, 1), col).float()

  def scatter_add_bwd(self, descs, n_inputs, batch, src_batch, grad_batch, grad_stride, src_ptrs,
                      grad_ptrs, rot, scale, scale_ptr, ids64, act_dtype, vec4, vec8, sync,
                      staged=False):
    self._count("scatter_add_bwd")
    self._wait(sync)
    if staged:  # the contract of the cp.async variant: 16-byte multiples / alignment everywhere
      esz = 4 if int(act_dtype) == 0 else 2
      assert (grad_stride * esz) % 16 == 0 and all(int(p) % 16 == 0 for p in grad_ptrs)
      for d in self._descs(descs, n_inputs):
        rb = int(d["width"]) * esz
        assert rb % 16 == 0 and rb <= 256 and (int(d["dst_col"]) * esz) % 16 == 0
    if scale_ptr:
      scale = scale * float(self.world.tensor(int(scale_ptr), torch.float32, 1, "lr")[0])
    for d in self._descs(descs, n_inputs):
      table = self._table(d)
      for dd in range(-(-batch // grad_batch)):
        g0, g1 = dd * grad_batch, min(batch, (dd + 1) * grad_batch)
        vals, lens = self._ids_of(d, g0, g1, ids64, src_ptrs, src_batch)
        ids = vals + int(d["id_shift"])
        ok = (ids >= 0) & (ids < int(d["sub_rows"]))
        g = self._grad_rows(d, dd, g1 - g0, grad_ptrs, grad_stride, act_dtype)
        w = torch.full((g1 - g0,), float(scale))
        if int(d["combiner"]) == 1:
          w = w / lens.clamp(min=1).to(w.dtype)
        per_id = (g * w.unsqueeze(1))[self._pool_index(lens)]
        table.index_add_(0, int(d["row_base"]) + ids[ok], per_id[ok])

  def sort_items(self, descs, tables, n_tables, n_inputs, batch, src_batch, src_ptrs, ids64,
                 n_items, total_rows, prefill_sentinel):
    self._count("sort_items")
    D = self._descs(descs, n_inputs)
    T = self._descs(tables, n_tables, TABLE_DESC)
    keys = torch.full((n_items,), int(total_rows), dtype=torch.int64)
    items = torch.zeros(n_items, dtype=torch.int64)
    covered = torch.zeros(n_items, dtype=torch.bool)
    for f, d in enumerate(D):
      vals, lens = self._ids_of(d, 0, batch, ids64, src_ptrs, src_batch)
      ids = vals + int(d["id_shift"])
      ok = (ids >= 0) & (ids < int(d["sub_rows"]))
      key = int(T[int(d["local_table"])]["key_base"]) + int(d["row_base"]) + ids
      key = torch.where(ok, key, torch.full_like(key, int(total_rows)))
      first = int(d["item_off"])
      if int(d["offsets"]):
        offs = self.world.tensor(int(d["offsets"]), torch.int64, batch + 1, "csr offsets")
        first += int(offs[0])
      n = key.numel()
      assert first + n <= n_items, "item range outside the sort buffers"
      assert not bool(covered[first:first + n].any()), "item ranges of two inputs overlap"
      covered[first:first + n] = True
      keys[first:first + n] = key
      items[first:first + n] = f * batch + self._pool_index(lens)
    if not prefill_sentinel:
      assert bool(covered.all()), "fixed-hotness inputs must fill the sort buffers exactly"
    order = torch.sort(keys, stable=True).indices
    ks, its = keys[order], items[order]
    heads = torch.ones(n_items, dtype=torch.bool)
    heads[1:] = ks[1:] != ks[:-1]
    starts = torch.nonzero(heads).view(-1)
    seg = torch.zeros(n_items + 1, dtype=torch.int64)
    seg[:starts.numel()] = starts
    seg[starts.numel()] = n_items
    return ks, its.to(torch.int32), seg, torch.tensor([starts.numel()], dtype=torch.int64)

  def segment_update(self, descs, tables, n_tables, batch, grad_batch, grad_stride, grad_ptrs,
                     keys, items, seg, n_unique, kind, lr, eps, beta1, beta2, bias1, bias2,
                     grad_scale, weight_decay, lr_ptr, emit_keys, emit_rows, max_width, act_dtype,
                     vec4, scratch, step_ptr, table_dtype=0):
    self._count("segment_update")
    tdt = self._ADT[int(table_dtype)]
    tsz = 4 if int(table_dtype) == 0 else 2
    step = 0
    # the kernels take the optimizer constants in fp32 and form 1 - beta and the bias
    # corrections in fp32 from them
    beta1, beta2 = float(np.float32(beta1)), float(np.float32(beta2))
    if step_ptr:
      t = float(self.world.tensor(int(step_ptr), torch.float32, 1, "optimizer step")[0])
      step = int(t)
      if kind == 3:
        bias1 = float(np.float32(1) - np.float32(beta1)**np.float32(t))
        bias2 = float(np.float32(1) - np.float32(beta2)**np.float32(t))
    D = self._descs(descs, 1 << 30)
    T = self._descs(tables, n_tables, TABLE_DESC)
    if lr_ptr:
      lr = float(self.world.tensor(int(lr_ptr), torch.float32, 1, "lr")[0])
    sentinel = int(T[-1]["key_base"]) + int(T[-1]["rows"])
    bases = [int(t["key_base"]) for t in T]
    gdt = self._ADT[int(act_dtype)]
    gsz = 4 if int(act_dtype) == 0 else 2
    nu = int(n_unique[0])
    for u in range(nu):
      k0, k1 = int(seg[u]), int(seg[u + 1])
      key = int(keys[k0])
      if key >= sentinel:
        if kind == 4:
          emit_keys[u] = sentinel
        continue
      m = max(i for i, b in enumerate(bases) if b <= key)
      t = T[m]
      width, row = int(t["width"]), key - bases[m]
      acc = torch.zeros(width)
      for k in range(k0, k1):
        item = int(items[k]) & 0xFFFFFFFF
        f, g = divmod(item, batch)
        d = D[f]
        assert int(d["local_table"]) == m and int(d["width"]) == width
        dd, i = divmod(g, grad_batch)
        w = 1.0
        if int(d["combiner"]) == 1:
          if int(d["offsets"]):
            o = self.world.tensor(int(d["offsets"]) + g * 8, torch.int64, 2, "csr offsets")
            w = 1.0 / float(int(o[1]) - int(o[0]))
          else:
            w = 1.0 / float(int(d["hotness"]))
        src = self.world.tensor(int(grad_ptrs[dd]) + (i * grad_stride + int(d["dst_col"])) * gsz,
                                gdt, width, "gradient source")
        acc += w * src.float()
      g = acc * grad_scale
      if kind == 4:
        emit_keys[u] = key
        emit_rows[u, :width] = g
        continue
      wt = self.world.tensor(int(t["weight"]) + row * width * tsz, tdt, width, "weight")
      if tsz == 2:
        # 16-bit table: fp32 math on an fp32 copy of the row, stochastic rounding back
        w16, wt = wt, wt.float()
      if weight_decay:
        g = g + weight_decay * wt
      if kind == 0:
        wt -= lr * g
      elif kind == 1:
        a = self.world.tensor(int(t["state0"]) + row * width * 4, torch.float32, width, "state0")
        a += g * g
        wt -= lr * g / (a.sqrt() + eps)
      elif kind == 2:
        a = self.world.tensor(int(t["state0"]) + row * 4, torch.float32, 1, "row state")
        a += (g * g).sum() / width
        wt -= lr * g / (a.sqrt() + eps)
      elif kind == 3:
        mm = self.world.tensor(int(t["state0"]) + row * width * 4, torch.float32, width, "adam m")
        vv = self.world.tensor(int(t["state1"]) + row * width * 4, torch.float32, width, "adam v")
        mm.mul_(beta1).add_(float(np.float32(1) - np.float32(beta1)) * g)
        vv.mul_(beta2).add_(float(np.float32(1) - np.float32(beta2)) * g * g)
        wt -= lr * (mm / bias1) / ((vv / bias2).sqrt() + eps)
      else:
        raise ValueError(f"optimizer kind {kind}")
      if tsz == 2:
        w16.copy_(stochastic_round(wt, tdt, step, key))


class DryRank:
  """What one simulated rank hands to its :class:`FusedEngine` (``FusedEngine(de, dry=...)``)."""

  def __init__(self, world: DryWorld, rank: int):
    self.ctx = DryCtx(world, rank)
    self.ops = world.make_ops(rank)

  def attach(self, engine):
    self.ops.engine = engine


def run_ranks(world: DryWorld, fn, timeout: float = 300.0):
  """Run ``fn(rank)`` for every rank in its own thread; re-raise the first failure."""
  results: List = [None] * world.world_size
  errors: List[Optional[BaseException]] = [None] * world.world_size

  def body(r):
    try:
      results[r] = world.run_rank(fn, r)
    except BaseException as e:  # pylint: disable=broad-except
      errors[r] = e
      world._barrier.abort()

  threads = [threading.Thread(target=body, args=(r,), daemon=True)
             for r in range(world.world_size)]
  # one intra-op thread per simulated rank: W Python threads each spawning a full OpenMP team
  # only oversubscribe the cores (the tensors are tiny)
  prev_threads = torch.get_num_threads()
  torch.set_num_threads(1)
  try:
    for t in threads:
      t.start()
    for t in threads:
      t.join(timeout)
  finally:
    torch.set_num_threads(prev_threads)
  real = [e for e in errors if e is not None and not isinstance(e, threading.BrokenBarrierError)]
  if real:
    raise real[0]
  if any(e is not None for e in errors) or any(t.is_alive() for t in threads):
    raise RuntimeError("a simulated rank hung or its barrier broke")
  return results


def build_engines(embeddings: Sequence[dict], world_size: int, world_cls=DryWorld, **kwargs):
  """One ``DistributedEmbedding`` + dry fused engine per rank of the plan (host memory).
  ``embeddings`` are config dicts; ``world_cls(world_size)`` makes the :class:`DryWorld`;
  ``kwargs`` go to ``DistributedEmbedding``."""
  from .dist_model_parallel import DistributedEmbedding  # pylint: disable=import-outside-toplevel
  assert world_size <= MAX_PEERS
  world = world_cls(world_size)
  des = []
  for r in range(world_size):
    de = DistributedEmbedding([dict(e) for e in embeddings], device="cpu", backend="torch",
                              world_size=world_size, rank=r, **kwargs)
    de.backend = "fused"
    de._bcast_hook = world.bcast
    de._barrier_hook = world.barrier
    de._engine = _fused.FusedEngine(de, dry=DryRank(world, r))
    des.append(de)
  return world, des

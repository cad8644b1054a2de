"""Fused execution engine of :class:`DistributedEmbedding` (CUDA, sm_90a).

Data flow of one training step on every rank (``W`` ranks, local batch ``b``, global ``B = W*b``).
Every exchange is a *push* over NVLink from inside a data kernel, and the cross-GPU ordering is
folded into those kernels (head waits / tail signals on peer-mapped flag words, ``SyncArgs`` in
``ops/csrc/de_b200.h``) - there is no separate barrier launch and no NCCL call on the hot path.

forward
  1. ids of all features are staged in ``in_flat`` (data loaders can write it directly, so the
     H2D copy is the staging);
  2. ``push_segments``: every rank stores the id segments of each feature straight into the id
     buffer of the rank that owns the feature (index all-to-all, reference DMP:211); its tail
     signals "ids ready";
  3. one descriptor-driven lookup kernel waits for the ids of all requesters, gathers + pools the
     rows of *all* local tables and stores every pooled row into the requester's ``out_buf`` at
     its final column offset (pooled-vector all-to-all + reorder + column-slice concat fused into
     the gather epilogue); its tail signals "output ready";
  4. the consumer of ``out_buf`` waits for that signal (a one-block kernel here, the head of the
     interaction kernel in the hand-scheduled DLRM step).
backward
  1. the producer of the gradient (``push_grad`` here, the interaction backward in the DLRM step)
     stores every piece of its gradient rows into the *owner's* receive buffer
     (``[B, sum(local widths)]``) and signals "gradient ready";
  2. the owner's update kernel waits for all requesters, reads the gradient rows from local
     memory and updates the tables in place: vector ``red.global.add`` (SGD), or the sorted /
     deduplicated path that sums each unique row once and applies SGD / Adagrad / row-wise
     Adagrad / Adam.  Its tail signals "consumed" so the next step's id push may overwrite.

Ragged (variable hotness) inputs keep the pull-style index exchange (the global CSR needs every
source's nnz): flag barrier + ``gather_segments`` / ``gather_ragged``.

Replaces ``_call_table_parallel`` / ``_call_row_slice`` / ``_call_data_parallel`` plus Horovod's
alltoall and the TF sparse optimizer kernels (reference dist_model_parallel.py:836-904).
"""
from __future__ import annotations

import os
import weakref
from typing import Any, Dict, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np
import torch

from ..ops import _native
from ..ops._native import DTYPE_CODE, GRAD_ROUTE, INPUT_DESC, TABLE_DESC
from ..ops.ragged import RaggedIds
from ..utils import nvtx
from .comm import CH_BARRIER0, CH_CONSUMED, CH_GRAD, CH_IDS, CH_OUT, CommContext
from .offload_cache import OffloadCache, split_budget

_OPT_KIND = {"sgd": _native.OPT_SGD, "adagrad": _native.OPT_ADAGRAD,
             "rowwise_adagrad": _native.OPT_ROWWISE_ADAGRAD, "adam": _native.OPT_ADAM}
_COMB = {None: 0, "sum": 0, "mean": 1}

# InputDesc.flags
FLAG_SKIP_EMPTY = 1   # store only when an id of the sample falls inside this shard
FLAG_CATCH_LOW = 2    # with SKIP_EMPTY: also store (zeros) when the shifted id is negative
FLAG_CATCH_HIGH = 4   # with SKIP_EMPTY: also store (zeros) when the shifted id >= sub_rows


def _weight(layer):
  return layer.embeddings


def _dev_ptr(t: torch.Tensor) -> int:
  """Device-visible address of a tensor: CUDA tensors directly, pinned host tensors (CPU
  offloaded tables / optimizer state) through their zero-copy UVA mapping."""
  if t.is_cuda:
    return t.data_ptr()
  if not t.is_pinned():
    raise RuntimeError("host-resident tables must live in pinned memory for the fused back end")
  return int(_native.require().host_device_pointer(t))


class ProducerUpdate(NamedTuple):
  """The SGD table update a gradient producer applies itself (:meth:`FusedEngine.producer_update`):
  one host InputDesc record per feature for ``ops.interact_bwd`` (null table: left to the
  scatter), the scale and learning-rate word of the update, and the descriptors of the tables the
  scatter still updates."""
  mpdesc: torch.Tensor       # the plan's model-parallel descriptors it was split from
  apply_descs: torch.Tensor
  scale: float
  scale_ptr: int
  ids64: bool
  rest_descs: Optional[torch.Tensor]
  n_rest: int

  def interact_args(self) -> tuple:
    """The trailing ``apply_*`` arguments of ``ops.interact_bwd``."""
    return self.apply_descs, self.scale, self.scale_ptr, self.ids64


class _FusedFn(torch.autograd.Function):

  @staticmethod
  def forward(ctx, engine, token, train, *weights):  # pylint: disable=arguments-differ
    ctx.engine = engine
    ctx.n_weights = len(weights)
    ctx.done = False
    engine._gen += 1
    ctx.gen = engine._gen
    out = engine._run_forward(train)
    # the backward of this call reads the engine's id / gradient buffers: remember the node so
    # that a second forward before this backward is routed elsewhere (see FusedEngine.busy)
    engine._pending = weakref.ref(ctx)
    if not getattr(engine.de, "zero_copy_output", False):
      out = out.clone()  # the engine buffer is overwritten by the next forward
    return out

  @staticmethod
  def backward(ctx, grad_out):  # pylint: disable=arguments-differ
    engine = ctx.engine
    if ctx.gen != engine._gen:
      raise RuntimeError(
          "DistributedEmbedding (fused back end): another forward ran on this layer before the "
          "backward of an earlier one; its index buffers were overwritten.  Call backward first, "
          "or use backend='torch' for several forwards per backward.")
    ctx.done = True
    grads = engine._run_backward(grad_out)
    return (None, None, None) + tuple(grads)


class FusedEngine:

  def __init__(self, de, dry=None):
    """``dry``: a :class:`dry_run.DryRank` - the engine then builds its descriptors against host
    buffers and runs them through the Python plan interpreter instead of the CUDA kernels (all
    ranks of a plan in one process, no GPU; see ``dry_run.py``)."""
    self.de = de
    self.st = de.strategy
    self.W, self.rank = de.world_size, de.rank
    self.device = de.device
    self.dry = dry is not None
    if self.dry:
      self.ops, self.ctx = dry.ops, dry.ctx
      dry.attach(self)
    else:
      self.ops = _native.require()
      self.ctx = CommContext.for_group(de.group, self.device)
    if self.W > 1 and not self.ctx.p2p:
      raise RuntimeError("fused back end needs CUDA peer access between all ranks")
    st = self.st
    imap = st.input_table_map
    self.out_widths = [int(st.global_configs[t]["output_dim"]) for t in imap]
    self.out_cols = [0]
    for w in self.out_widths:
      self.out_cols.append(self.out_cols[-1] + w)
    self.total_width = self.out_cols[-1]
    self.compute_dtype = de.compute_dtype
    if self.compute_dtype not in DTYPE_CODE:
      raise ValueError("fused back end supports fp32, bf16 and fp16 activations")
    self.act = DTYPE_CODE[self.compute_dtype]  # dtype code of activations / gradients on the wire
    # storage of the model-parallel tables (one dtype for all of them); replicated tables are fp32
    self.table_dtype = getattr(de, "table_dtype", torch.float32)
    self.tab = DTYPE_CODE[self.table_dtype]
    self._key = None
    self._gen = 0          # forward generation (see _FusedFn)
    self._pending = None   # weakref to the autograd node of the last forward
    self._token = torch.zeros((), device=self.device)
    self.lr_t = torch.zeros(1, dtype=torch.float32, device=self.device)
    self._lr_external = False  # True once a trainer aliases lr_t with its own device word
    # Adam step count, device resident so that a captured CUDA graph keeps advancing it
    self.step_t = torch.zeros(1, dtype=torch.float32, device=self.device)
    self.opt_state: Dict[int, List[torch.Tensor]] = {}
    self._tables_dirty = True
    self._dp_targets = None
    self._dp_target_desc = None
    self.out_row_stride = None  # see set_out_row_stride
    self.push_chunk_rows = None  # see enable_streamed_push
    self._dry_updates = False   # see dry_updates()
    # local model-parallel tables: table-parallel first, then row slices
    self.mp_layers = list(de.local_embedding_layers) + list(de.row_layers)
    self.n_col_tables = len(de.local_embedding_layers)
    # host-resident tables are read zero-copy over PCIe; their update must not use atomics
    self.has_offload = any(getattr(l, "cpu_offloaded", False) for l in self.mp_layers)
    # HBM row cache of the offloaded table-parallel tables (offload_cache.py), local table -> cache
    self.cache_size = getattr(de, "offload_cache_size", None)
    self.caches: Dict[int, OffloadCache] = {}
    self._cache_plan: List[tuple] = []
    if self.cache_size is not None and (self.dry or self.W > 1):
      raise NotImplementedError("the offload cache runs on one rank (world size 1) for now")

  def _ptr(self, t: torch.Tensor) -> int:
    return t.data_ptr() if self.dry else _dev_ptr(t)

  def _sync(self, wait: int = -1, wait_abs: int = -1, signal: int = -1):
    return self.ctx.sync(wait=wait, wait_abs=wait_abs, signal=signal) if self.W > 1 else []

  def dry_updates(self, on: bool):
    """While on, the update kernels run on a zero gradient (scale 0) without weight decay and the
    optimizer step counter is left alone: the warm-up passes a trainer runs before capturing its CUDA graph
    exercise every kernel (lazy module loading, workspaces) without touching the tables or the
    optimizer state (Adagrad accumulators would otherwise absorb the warm-up gradients)."""
    self._dry_updates = bool(on)

  def enable_streamed_push(self, chunk_rows: Optional[int]):
    """Gradient all-to-all through a local staging buffer + a streaming copy kernel.

    A fused producer (the DLRM interaction backward) that stores its gradient pieces straight
    into peer memory is throttled by NVLink back-pressure on its own load/store pipe: compute
    and transfer serialise, well below the rate a pure copy kernel reaches.
    With this on, the producer writes the pieces of remote owners into ``gstage`` (owner-major,
    local memory, ``routes_stage``) and counts finished rows per chunk of ``chunk_rows``
    samples; :meth:`launch_streamed_push` runs a small copy kernel next to it that forwards
    every finished chunk to its owner and signals "gradient ready" at the end."""
    if chunk_rows != self.push_chunk_rows:
      self.push_chunk_rows = chunk_rows
      if self._key is not None:
        self.close()

  def set_out_row_stride(self, stride: Optional[int]):
    """Row stride (elements, multiple of 8) of the output buffer, >= sum of the output widths.
    A consumer that concatenates the embeddings with other features (the synthetic models' MLP
    input) lets the lookups write straight into its input matrix: ``out_full`` is the whole
    ``[batch, stride]`` buffer, ``out`` the ``[batch, sum(widths)]`` view of its first columns."""
    if stride is not None and (stride < self.total_width or stride % 8):
      raise ValueError("out row stride must be a multiple of 8 and >= the total output width")
    if stride != self.out_row_stride:
      self.out_row_stride = stride
      if self._key is not None:
        self.close()

  # ------------------------------------------------------------------ capabilities
  def busy(self) -> bool:
    """True while a forward that recorded an autograd graph has not run its backward (and the
    graph is still alive): the engine's id / output / gradient buffers belong to that call, so a
    further forward must not run on the engine (the caller falls back to the torch back end;
    the reference layer can be called any number of times)."""
    node = self._pending() if self._pending is not None else None
    return node is not None and not node.done

  def supports(self, inputs) -> bool:
    st, de = self.st, self.de
    col_inputs = set(st.input_groups[1]) if de.dp_input else set(range(len(inputs)))
    imap = st.input_table_map
    for i, x in enumerate(inputs):
      if isinstance(x, RaggedIds):
        if i not in col_inputs:  # ragged only for table-parallel features
          return False
        continue
      if not isinstance(x, torch.Tensor) or x.dim() > 2:
        return False
      if x.dim() == 2 and x.shape[1] != 1:
        # the kernels always pool a sample's ids: a table without a combiner keeps them apart
        # ([b, h, width]) -> torch back end for every group (table parallel, replicated, row)
        t = imap[i] if de.dp_input else \
            st.table_groups[1][st.map_groups[1][st.input_ids_list[self.rank][i]]]
        if st.global_configs[t].get("combiner") is None:
          return False
    return True

  # ------------------------------------------------------------------ plan -> layouts
  def _mp_layout(self, r: int, hots: Optional[Tuple[int, ...]], B: int):
    """Owner-side layout of rank ``r``: item offsets of its local inputs in the id buffer
    (needs the hotness of every input: dp_input mode, or ``r`` = this rank) and their column
    offsets / widths in its gradient receive buffer.  Every rank computes every rank's layout
    from the global plan."""
    de, st = self.de, self.st
    col_group = st.input_groups[1]
    col_map = st.map_groups[1]
    my_inputs = st.input_ids_list[r] if st.table_groups[1] else []
    items, cols, widths, pos, col = [], [], [], 0, 0
    for li, k in enumerate(my_inputs):
      shard = next(s for s in st.shards[r] if s.table == col_map[k])
      if hots is not None:
        gi = col_group[k] if de.dp_input else li
        items.append(pos)
        pos += B * abs(hots[gi])
      cols.append(col)
      widths.append(int(shard.width))
      col += int(shard.width)
    row_inputs = st.input_groups[2] if de.dp_input else []
    for j, gi in enumerate(row_inputs):
      m = st.map_groups[2][j]
      w = int(st.row_sliced_configs[r][m]["output_dim"])
      if hots is not None:
        items.append(pos)
        pos += B * abs(hots[gi])
      cols.append(col)
      widths.append(w)
      col += w
    return {"items": items, "n_items": pos, "cols": cols, "widths": widths, "width": col,
            "n_col": len(my_inputs)}

  # ------------------------------------------------------------------ buffer lifecycle
  _SYM_BUFS = ("in_buf", "split_buf", "ids_buf", "out_buf", "recv_buf", "rs_buf")
  _SYM_VIEWS = ("in_flat", "in_views", "split_flat", "split_views", "ids_mp", "out", "out_full",
                "recv", "rs", "gstage")

  def close(self):
    """Release the symmetric buffers (collective: every rank of the group must call it at the
    same point).  Peer mappings are closed on *all* ranks before any rank frees its memory -
    otherwise a later cudaMalloc may hand the freed address out again while a peer still maps
    it, and the next IPC open of that address fails ("resource already mapped")."""
    bufs = [getattr(self, n, None) for n in self._SYM_BUFS]
    bufs = [b for b in bufs if b is not None]
    if bufs and self.W > 1 and not self.dry:
      torch.cuda.synchronize(self.device)
      for b in bufs:
        b.close()
      torch.distributed.barrier(group=self.de.group)
    for n in self._SYM_BUFS + self._SYM_VIEWS:
      if hasattr(self, n):
        setattr(self, n, None)
    self._key = None

  # ------------------------------------------------------------------ plan -> descriptors
  def _build(self, b: int, hots: Tuple[int, ...], ids64: bool):
    de, st, W, rank = self.de, self.st, self.W, self.rank
    dev = self.device
    if self._key is not None:
      self.close()  # new batch size / hotness: the old symmetric buffers go first
    id_dtype = torch.int64 if ids64 else torch.int32
    idsz = 8 if ids64 else 4
    B = b * W if de.dp_input else b
    lb = b if de.dp_input else b // W  # local (requester) batch
    self.B, self.lb, self.hots, self.ids64, self.id_dtype = B, lb, hots, ids64, id_dtype
    csz = 4 if self.act == 0 else 2

    col_group = st.input_groups[1] if de.dp_input else list(range(len(hots)))
    col_map = st.map_groups[1]
    # --- staging of data-parallel inputs
    # hots[i] > 0: fixed hotness; hots[i] < 0: ragged input with capacity -hots[i] ids per sample
    self.ragged = [h < 0 for h in hots]
    self.any_ragged = any(self.ragged)
    n_rag = sum(self.ragged)
    rag_index = {}
    for i, r in enumerate(self.ragged):
      if r:
        rag_index[i] = len(rag_index)
    # index exchange: "push" (fire-and-forget stores into the owners' id buffers, signalling
    # folded into the kernels) unless a ragged input needs the pull-style global CSR build
    self.id_mode = "none" if W == 1 or not de.dp_input else ("pull" if self.any_ragged else "push")
    if de.dp_input:
      in_off, pos = [], 0
      for h in hots:
        in_off.append(pos)
        pos += b * abs(h)
      self.in_elems = max(pos, 1)
      if self.id_mode == "pull":
        self.in_buf = self.ctx.alloc(self.in_elems * idsz, "ids_in")
        in_flat = self.in_buf.view(id_dtype, (self.in_elems,))
        self.in_ptrs = self.in_buf.peer_ptrs()
      else:
        self.in_buf = None
        in_flat = torch.zeros(self.in_elems, dtype=id_dtype, device=dev)
        self.in_ptrs = [in_flat.data_ptr()]
      self.in_flat = in_flat
      self.in_views = [in_flat[o:o + b * abs(h)].view(b, abs(h)) for o, h in zip(in_off, hots)]
      # row_splits of ragged inputs (int64, [b + 1] each) live in their own symmetric buffer
      if n_rag:
        n_sp = n_rag * (b + 1)
        if W > 1:
          self.split_buf = self.ctx.alloc(n_sp * 8, "ragged_splits")
          self.split_flat = self.split_buf.view(torch.int64, (n_sp,))
          self.split_ptrs = self.split_buf.peer_ptrs()
        else:
          self.split_buf = None
          self.split_flat = torch.zeros(n_sp, dtype=torch.int64, device=dev)
          self.split_ptrs = [self.split_flat.data_ptr()]
        self.split_views = {i: self.split_flat[j * (b + 1):(j + 1) * (b + 1)]
                            for i, j in rag_index.items()}
    else:
      in_off = None
      self.in_buf, self.in_flat, self.in_views, self.in_ptrs = None, None, None, []
      self.split_views = {}

    # --- owner-side layouts of every rank (id buffer items, gradient receive columns)
    layouts = [self._mp_layout(r, hots if (de.dp_input or r == rank) else None, B)
               for r in range(W)]
    mine = layouts[rank]
    my_inputs = st.input_ids_list[rank] if st.table_groups[1] else []
    row_inputs = st.input_groups[2] if de.dp_input else []
    n_col, n_row = len(my_inputs), len(row_inputs)
    col_items, row_items = mine["items"][:n_col], mine["items"][n_col:]
    self.n_items = mine["n_items"]
    self.recv_width = max(mine["width"], 1)
    need_copy = (W > 1) or (not de.dp_input)
    # model-parallel id buffer (global batch of every local input); peers store into it
    if self.id_mode == "push":
      n_sym = max(max(l["n_items"] for l in layouts), 1)
      self.ids_buf = self.ctx.alloc(n_sym * idsz, "ids_mp")
      self.ids_mp = self.ids_buf.view(id_dtype, (n_sym,))
      self.ids_ptrs = self.ids_buf.peer_ptrs()
    else:
      self.ids_buf = None
      self.ids_mp = torch.zeros(max(self.n_items, 1), dtype=id_dtype, device=dev) \
          if need_copy else None
      self.ids_ptrs = []
    # global-batch CSR offsets of the ragged local inputs ([B + 1] each)
    my_ragged = [li for li, k in enumerate(my_inputs)
                 if self.ragged[col_group[k] if de.dp_input else li]]
    self.goff = torch.zeros(max(len(my_ragged) * (B + 1), 1), dtype=torch.int64, device=dev)
    goff_index = {li: j for j, li in enumerate(my_ragged)}

    def ids_ptr(item_off, gi):
      if need_copy:
        return self.ids_mp.data_ptr() + item_off * idsz
      return self.in_flat.data_ptr() + in_off[gi] * idsz

    # --- table descriptors (sorted-update path)
    self._make_caches(B, hots, col_group, my_inputs, col_items)
    tdesc = np.zeros(len(self.mp_layers), dtype=TABLE_DESC)
    key = 0
    for m, layer in enumerate(self.mp_layers):
      w = _weight(layer)
      rows = self.caches[m].slots if m in self.caches else w.shape[0]
      tdesc[m]["weight"] = self._ptr(w)
      tdesc[m]["rows"] = rows
      tdesc[m]["key_base"] = key
      tdesc[m]["width"] = w.shape[1]
      key += rows
    self.total_rows = key
    self.tdesc_np = tdesc
    self.max_width = max([int(_weight(l).shape[1]) for l in self.mp_layers] + [1])

    # --- output buffer (requester side) and gradient receive buffer (owner side)
    tw = self.total_width
    ostride = self.out_stride = int(self.out_row_stride or tw)
    out_bytes = max(lb * ostride * csz, 16)
    recv_w_sym = max(max(l["width"] for l in layouts), 1)
    if W > 1:
      self.out_buf = self.ctx.alloc(out_bytes, "emb_out")
      self.out_full = self.out_buf.view(self.compute_dtype, (lb, ostride))
      self.out = self.out_full[:, :tw]
      self.out_ptrs = self.out_buf.peer_ptrs()
      self.recv_buf = self.ctx.alloc(max(B * recv_w_sym * csz, 16), "emb_grad_recv")
      self.recv = self.recv_buf.view(self.compute_dtype, (B, self.recv_width))
      recv_ptrs = self.recv_buf.peer_ptrs()
    else:
      self.out_buf = self.recv_buf = None
      self.out_full = torch.zeros(lb, ostride, dtype=self.compute_dtype, device=dev)
      self.out = self.out_full[:, :tw]
      self.out_ptrs = [self.out.data_ptr()]
      self.recv = torch.zeros(B, self.recv_width, dtype=self.compute_dtype, device=dev)
      recv_ptrs = [self.recv.data_ptr()]
    self.recv_ptr = [self.recv.data_ptr()]
    # requester-layout gradient of the replicated inputs (written by a fused producer such as
    # the DLRM interaction backward; the generic path reads the incoming gradient directly)
    dp_inputs = st.input_groups[0] if de.dp_input else []
    self.grad = torch.zeros(lb, tw, dtype=self.compute_dtype, device=dev) if len(dp_inputs) \
        else None

    # --- table-parallel descriptors
    pieces = {(p.rank, p.local_input): p for p in st.output_pieces}
    cdesc = np.zeros(n_col, dtype=INPUT_DESC)
    segs, rsegs = [], []      # pull mode: what this rank fetches
    for li, k in enumerate(my_inputs):
      gi = col_group[k] if de.dp_input else li
      t_in_group = col_map[k]
      shard = next(s for s in st.shards[rank] if s.table == t_in_group)
      layer = de.local_embedding_layers[shard.local_table]
      w = _weight(layer)
      d = cdesc[li]
      d["table"] = self._ptr(w)
      d["ids"] = ids_ptr(col_items[li], gi)
      d["ids_off"] = 0
      d["sub_rows"] = shard.rows
      d["row_base"] = shard.row_offset
      d["width"] = shard.width
      d["hotness"] = max(hots[gi], 0)
      if self.ragged[gi]:
        if need_copy:
          d["offsets"] = self.goff.data_ptr() + goff_index[li] * (B + 1) * 8
        else:  # single rank, dp input: the staged CSR is already the global one
          d["offsets"] = self.split_views[gi].data_ptr()
      gi_global = st.input_groups[1][k]
      d["dst_col"] = self.out_cols[gi_global] + pieces[(rank, li)].col_offset
      d["combiner"] = _COMB[layer.combiner]
      d["local_table"] = shard.local_table
      d["item_off"] = col_items[li]
      if layer.combiner is None and hots[gi] != 1:
        raise ValueError("table-parallel lookups without a combiner need one id per sample")
      if self.id_mode == "pull":
        if self.ragged[gi]:
          rsegs.append([in_off[gi], col_items[li], rag_index[gi] * (b + 1),
                        goff_index[li] * (B + 1)])
        else:
          for s in range(W):
            segs.append([s, in_off[gi], col_items[li] + s * b * hots[gi], b * hots[gi]])
    self._cache_descs(cdesc, col_items, B, hots, col_group, my_inputs, id_dtype)
    self.cdesc_np = cdesc

    # --- row-slice descriptors.  One-hot inputs: exactly one rank owns a sample's id, it stores
    # the row straight into the requester's output (rank 0 / the last rank also catch ids below /
    # above the table and store zeros).  Multi-hot inputs: every rank stores its partial pool
    # into slot `rank` of the requester's partial buffer, the requester sums the W slots.
    rdesc = np.zeros(n_row, dtype=INPUT_DESC)
    self.rs_width = 0
    self.rs_cols = []     # multi-hot row inputs: (gi, partial col, width)
    self.row_onehot = []
    for j, gi in enumerate(row_inputs):
      m = st.map_groups[2][j]
      layer = de.row_layers[m]
      w = _weight(layer)
      d = rdesc[j]
      d["table"] = w.data_ptr()
      d["ids"] = ids_ptr(row_items[j], gi)
      d["id_shift"] = st.row_inputs_offsets[rank][m]
      d["sub_rows"] = w.shape[0]
      d["width"] = w.shape[1]
      d["hotness"] = hots[gi]
      d["combiner"] = _COMB[layer.combiner]
      d["local_table"] = self.n_col_tables + m
      d["item_off"] = row_items[j]
      onehot = hots[gi] == 1
      self.row_onehot.append(onehot)
      if onehot:
        d["dst_col"] = self.out_cols[gi]
        d["flags"] = FLAG_SKIP_EMPTY | (FLAG_CATCH_LOW if rank == 0 else 0) | \
            (FLAG_CATCH_HIGH if rank == W - 1 else 0)
      else:
        d["dst_col"] = self.rs_width
        d["flags"] = 0
        self.rs_cols.append((gi, self.rs_width, int(w.shape[1])))
        self.rs_width += int(w.shape[1])
      if self.id_mode == "pull":
        for s in range(W):
          segs.append([s, in_off[gi], row_items[j] + s * b * hots[gi], b * hots[gi]])
    self.rdesc_np = rdesc
    oh = np.array(self.row_onehot, dtype=bool) if n_row else np.zeros(0, dtype=bool)
    # forward launches: [table-parallel + one-hot row inputs] -> out_buf; multi-hot rows -> rs_buf
    self.fwd_main_np = np.concatenate([cdesc, rdesc[oh]]) if n_row else cdesc
    self.fwd_rs_np = rdesc[~oh] if n_row else rdesc
    if len(self.fwd_rs_np):
      self.rs_buf = self.ctx.alloc(W * lb * self.rs_width * 4, "row_slice_partials")
      self.rs = self.rs_buf.view(torch.float32, (W, lb, self.rs_width))
      self.rs_ptrs = self.rs_buf.peer_ptrs(rank * lb * self.rs_width * 4)
      self.rs_cols_t = torch.tensor([[c0, self.out_cols[gi], w] for gi, c0, w in self.rs_cols],
                                    dtype=torch.int32, device=dev)
    else:
      self.rs_buf = None

    # --- replicated tables: plain local lookup of the local batch
    ddesc = np.zeros(len(dp_inputs), dtype=INPUT_DESC)
    for j, gi in enumerate(dp_inputs):
      m = st.map_groups[0][j]
      layer = de.dp_layers[m]
      w = _weight(layer)
      d = ddesc[j]
      d["table"] = w.data_ptr()
      d["ids"] = self.in_flat.data_ptr() + in_off[gi] * idsz
      d["sub_rows"] = w.shape[0]
      d["width"] = w.shape[1]
      d["hotness"] = hots[gi]
      d["dst_col"] = self.out_cols[gi]
      d["combiner"] = _COMB[layer.combiner]
      d["local_table"] = m
    self.ddesc_np = ddesc
    # persistent dense-gradient buffers of the replicated tables (generic autograd path)
    self._dp_grad_flat, self._dp_grad_views, self._dp_grad_desc = None, [], None
    self._dp_grad_desc_np = None
    if len(de.dp_layers):
      offs, pos = [], 0
      for layer in de.dp_layers:
        offs.append(pos)
        pos += (_weight(layer).numel() + 3) // 4 * 4
      self._dp_grad_flat = torch.zeros(max(pos, 4), dtype=torch.float32, device=dev)
      self._dp_grad_views = [self._dp_grad_flat[o:o + _weight(l).numel()].view(_weight(l).shape)
                             for o, l in zip(offs, de.dp_layers)]
      dd = ddesc.copy()
      for j in range(len(dd)):
        dd[j]["table"] = self._dp_grad_views[int(dd[j]["local_table"])].data_ptr()
      self._dp_grad_desc_np = dd

    # --- index push: what this rank sends ({dst rank, src offset, dst offset, n} per segment)
    push = []
    if self.id_mode == "push":
      for r in range(W):
        L = layouts[r]
        r_inputs = st.input_ids_list[r] if st.table_groups[1] else []
        for li, k in enumerate(r_inputs):
          gi = col_group[k]
          n = b * hots[gi]
          push.append([r, in_off[gi], L["items"][li] + rank * n, n])
        for j, gi in enumerate(row_inputs):
          n = b * hots[gi]
          push.append([r, in_off[gi], L["items"][L["n_col"] + j] + rank * n, n])
    self.push_segs = torch.tensor(push, dtype=torch.int64, device=dev) if push else None
    self.max_push = max([s[3] for s in push]) if push else 0

    # --- gradient routes: where every piece of this requester's gradient row goes
    # streamed push (enable_streamed_push): pieces of remote owners are staged locally,
    # owner-major, and forwarded by a copy kernel; every row must be a 16-byte multiple
    self.gstage, self.push_plan, self.push_counters = None, None, None
    stage_base = {}
    if self.push_chunk_rows and W > 1 and \
        all((layouts[r]["width"] * csz) % 16 == 0 for r in range(W)):
      offs, pos = {}, 0
      for r in range(W):
        if r != rank and layouts[r]["width"]:
          offs[r] = pos
          pos += (lb * layouts[r]["width"] * csz + 255) // 256 * 256
      self.gstage = torch.empty(max(pos, 256), dtype=torch.uint8, device=dev)
      stage_base = {r: self.gstage.data_ptr() + o for r, o in offs.items()}
      peers = sorted(offs, key=lambda r: (r - rank) % W)  # start with the next rank: spread ingress
      self.push_plan = ([stage_base[r] for r in peers],
                        [recv_ptrs[r] + rank * lb * layouts[r]["width"] * csz for r in peers],
                        [layouts[r]["width"] * csz for r in peers])
      n_chunks = -(-lb // self.push_chunk_rows)
      self.push_counters = torch.zeros(n_chunks, dtype=torch.int32, device=dev)
    routes, routes_stage = [], []
    for r in range(W):
      L = layouts[r]
      base = recv_ptrs[r] + rank * lb * L["width"] * csz
      sbase = stage_base.get(r, base)
      r_inputs = st.input_ids_list[r] if st.table_groups[1] else []
      for li, k in enumerate(r_inputs):
        p = pieces[(r, li)]
        gi_global = st.input_groups[1][k]
        item = (self.out_cols[gi_global] + p.col_offset, L["widths"][li], base, L["width"],
                L["cols"][li])
        routes.append(item)
        routes_stage.append(item[:2] + (sbase,) + item[3:])
      for j, gi in enumerate(row_inputs):
        item = (self.out_cols[gi], L["widths"][L["n_col"] + j], base, L["width"],
                L["cols"][L["n_col"] + j])
        routes.append(item)
        routes_stage.append(item[:2] + (sbase,) + item[3:])
    dp_routes = [(self.out_cols[gi], self.out_widths[gi], self.grad.data_ptr(), tw,
                  self.out_cols[gi]) for gi in dp_inputs]

    def pack(rs):
      rs = sorted(rs, key=lambda x: (x[0], x[2]))
      arr = np.zeros(len(rs), dtype=GRAD_ROUTE)
      for i, (src_col, width, dst, stride, dst_col) in enumerate(rs):
        arr[i]["dst"], arr[i]["dst_stride"] = dst, stride
        arr[i]["src_col"], arr[i]["width"], arr[i]["dst_col"] = src_col, width, dst_col
      return arr
    self.routes_mp_np = pack(routes)
    self.routes_all_np = pack(routes + dp_routes)
    self.routes_stage_np = pack(routes_stage + dp_routes) if self.gstage is not None else None

    self.segs = torch.tensor(segs, dtype=torch.int64, device=dev) if segs else None
    self.max_seg = max([s[3] for s in segs]) if segs else 0
    self.rsegs = torch.tensor(rsegs, dtype=torch.int64, device=dev) if rsegs else None
    self.max_rcap = b * max([abs(h) for h, r in zip(hots, self.ragged) if r] + [0])
    self.my_ragged_mp = my_ragged if not de.dp_input else []
    self.col_items = col_items
    # backward descriptors of all model-parallel inputs: gradient columns of the receive buffer
    mp = np.concatenate([cdesc, rdesc]) if n_row else cdesc.copy()
    for i in range(len(mp)):
      mp[i]["dst_col"] = mine["cols"][i]
    self.mpdesc_np = mp
    self.n_mp_inputs = len(mp)

    widths = [int(x) for x in list(cdesc["width"]) + list(rdesc["width"]) + list(ddesc["width"])]
    cols = [int(x) for x in list(self.fwd_main_np["dst_col"]) + list(self.fwd_rs_np["dst_col"]) +
            list(ddesc["dst_col"]) + list(mp["dst_col"])]
    self.vec4 = all(w % 4 == 0 for w in widths) and all(c % 4 == 0 for c in cols) and \
        tw % 4 == 0 and self.rs_width % 4 == 0 and self.recv_width % 4 == 0 and ostride % 4 == 0
    # 16-bit tables: 8 columns (one 16-byte load) per lane in the model-parallel lookups
    fw = [int(x) for x in list(self.fwd_main_np["width"]) + list(self.fwd_rs_np["width"])]
    fc = [int(x) for x in list(self.fwd_main_np["dst_col"]) + list(self.fwd_rs_np["dst_col"])]
    self.fwd_vec8 = self.tab != 0 and self.vec4 and all(w % 8 == 0 for w in fw) and \
        all(c % 8 == 0 for c in fc) and ostride % 8 == 0 and self.rs_width % 8 == 0
    # 16-byte gradient loads (8 columns per lane) in the SGD update: DE_B200_VEC8_GRAD=1
    self.vec8 = os.environ.get("DE_B200_VEC8_GRAD", "0") == "1" and self.vec4 and \
        all(w % 8 == 0 for w in widths) and all(c % 8 == 0 for c in cols) and \
        self.recv_width % 8 == 0
    # staged SGD update (gradient rows streamed through shared memory with cp.async): every
    # model-parallel gradient row must be a 16-byte multiple of at most 256 bytes, 16-byte aligned
    mpw = [int(x) for x in mp["width"]]
    mpc = [int(x) for x in mp["dst_col"]]
    self.staged_update = os.environ.get("DE_B200_SCATTER_STAGED", "1") == "1" and self.vec4 and \
        len(mp) > 0 and all((w * csz) % 16 == 0 and w * csz <= 256 for w in mpw) and \
        all((c * csz) % 16 == 0 for c in mpc) and (self.recv_width * csz) % 16 == 0
    # same for the requester-layout gradient of the replicated tables (fast-step path)
    self.staged_dp = os.environ.get("DE_B200_SCATTER_STAGED", "1") == "1" and self.vec4 and \
        len(ddesc) > 0 and (tw * csz) % 16 == 0 and \
        all((int(w) * csz) % 16 == 0 and int(w) * csz <= 256 for w in ddesc["width"]) and \
        all((int(c) * csz) % 16 == 0 for c in ddesc["dst_col"])
    self._upload()
    self._key = (b, hots, ids64)

  # ------------------------------------------------------------------ offload cache
  def _make_caches(self, B, hots, col_group, my_inputs, col_items):
    """(Re)create the caches of the offloaded tables for this batch layout; a cache whose spill
    region no longer fits is flushed to the host first."""
    if self.cache_size is None:
      return
    de = self.de
    cached = [m for m in range(self.n_col_tables) if getattr(self.mp_layers[m], "cpu_offloaded",
                                                             False)]
    n_spill = {m: 0 for m in cached}
    for li, k in enumerate(my_inputs):
      m = next(s for s in self.st.shards[self.rank]
               if s.table == self.st.map_groups[1][k]).local_table
      if m in n_spill:
        gi = col_group[k] if de.dp_input else li
        n_spill[m] += B * abs(hots[gi])
    cached = [m for m in cached if n_spill[m] > 0]
    # a table no input of this layout reads keeps no cache: its rows go back to the host
    for m in [m for m in self.caches if m not in cached]:
      self.caches.pop(m).flush(self.ops)
    sets = split_budget(int(self.cache_size),
                        [tuple(_weight(self.mp_layers[m]).shape) for m in cached])
    for m, n_sets in zip(cached, sets):
      old = self.caches.get(m)
      if old is not None and (old.n_sets, old.n_spill) == (n_sets, n_spill[m]):
        continue
      if old is not None:
        # a new batch size or hotness changes the spill region: the cache starts over.  The old
        # one is flushed and released before the new one is allocated (the flush is ordered
        # before any reuse of its memory by the stream), so the peak stays one cache per table
        self.caches.pop(m).flush(self.ops)
        del old
      c = OffloadCache(_weight(self.mp_layers[m]), n_sets, n_spill[m], self.device, self._ptr)
      if self.opt_state.get(m):
        c.set_state(self.opt_state[m])
      self.caches[m] = c

  def _cache_descs(self, cdesc, col_items, B, hots, col_group, my_inputs, id_dtype):
    """Point the cached inputs at the cache: their ids become slot ids in ``ids_cache`` (laid out
    like the owner's id buffer), their table the cache's weight rows.  Builds one pass plan per
    cached table from the original (host-row) descriptors."""
    self._cache_plan = []
    self.ids_cache = None
    if not self.caches:
      return
    dev = self.device
    self.ids_cache = torch.full((max(self.n_items, 1),), -1, dtype=id_dtype, device=dev)
    idsz = self.ids_cache.element_size()
    tab = np.zeros(1, dtype=TABLE_DESC)
    for m, c in self.caches.items():
      lis = [li for li in range(len(cdesc)) if int(cdesc[li]["local_table"]) == m]
      src = cdesc[lis].copy()
      remap = np.zeros(len(lis), dtype=_native.CACHE_REMAP)
      pos = 0
      for j, li in enumerate(lis):
        k = my_inputs[li]
        n = B * abs(hots[col_group[k] if self.de.dp_input else li])
        src[j]["local_table"] = 0
        src[j]["item_off"] = pos
        pos += n
        r = remap[j]
        r["ids"], r["n"] = cdesc[li]["ids"], n
        r["id_shift"], r["sub_rows"] = cdesc[li]["id_shift"], cdesc[li]["sub_rows"]
        r["row_base"], r["out_off"] = cdesc[li]["row_base"], col_items[li]
        d = cdesc[li]
        d["table"] = c.weight.data_ptr()
        d["ids"] = self.ids_cache.data_ptr() + col_items[li] * idsz
        d["id_shift"], d["row_base"], d["sub_rows"] = 0, 0, c.slots
      t = tab.copy()
      t[0]["rows"], t[0]["width"], t[0]["key_base"] = c.rows, c.width, 0
      t[0]["weight"] = self._ptr(c.host_weight)
      prefill = bool(src["offsets"].any())
      self._cache_plan.append((m, _native.upload_struct_array(src, dev),
                               _native.upload_struct_array(t, dev), len(src), pos, prefill,
                               _native.upload_struct_array(remap, dev), len(remap),
                               int(remap["n"].max())))

  def _run_cache_pass(self, train: bool):
    for m, descs, table, n_in, n_items, prefill, remap, n_remap, max_n in self._cache_plan:
      c = self.caches[m]
      self.ops.offload_cache_pass(c.tensors(), c.host_ptrs(), c.n_sets, c.n_spill, c.rows, descs,
                                  table, n_in, self.B, self.ids64, n_items, prefill, remap,
                                  n_remap, max_n, self.ids_cache.data_ptr(), bool(train))

  def flush_offload_cache(self, invalidate: bool = False):
    """Write every dirty cached row and its optimizer state back to the host tables (and, with
    ``invalidate``, empty the caches).  Synchronises the device: the host tables are final when
    this returns."""
    if not self.caches:
      return
    for c in self.caches.values():
      c.flush(self.ops)
      if invalidate:
        c.invalidate()
    torch.cuda.synchronize(self.device)

  def offload_cache_stats(self, reset: bool = True) -> Dict[int, Dict[str, int]]:
    return {m: c.read_stats(reset) for m, c in self.caches.items()}

  def _upload(self):
    """(Re)upload descriptor arrays; table pointers / optimizer state may have changed."""
    dev = self.device
    up = _native.upload_struct_array
    self.fwd_main = up(self.fwd_main_np, dev) if len(self.fwd_main_np) else None
    self.fwd_rs = up(self.fwd_rs_np, dev) if len(self.fwd_rs_np) else None
    # forward launches of the main group: (descs, n, samples per warp tile).  One-hot / low
    # hotness inputs use 32-sample tiles; inputs that pool many rows per sample go into a second
    # launch with small tiles (~64 gathered rows per tile) so that long segments spread over
    # many warps instead of one warp walking 32 long samples
    self.fwd_launches = []
    if len(self.fwd_main_np):
      hot = self._desc_hotness(self.fwd_main_np)
      low = hot <= 4
      for mask in (low, ~low):
        if mask.any():
          d = self.fwd_main_np[mask]
          self.fwd_launches.append((up(d, dev), int(mask.sum()), self._tile_samples(d, hot[mask])))
    self.fwd_rs_tile = self._tile_samples(self.fwd_rs_np, self._desc_hotness(self.fwd_rs_np)) \
        if len(self.fwd_rs_np) else 32
    self.ddesc = up(self.ddesc_np, dev) if len(self.ddesc_np) else None
    self.mpdesc = up(self.mpdesc_np, dev) if len(self.mpdesc_np) else None
    self.routes_mp = up(self.routes_mp_np, dev) if len(self.routes_mp_np) else None
    self.routes_all = up(self.routes_all_np, dev) if len(self.routes_all_np) else None
    self.routes_stage = up(self.routes_stage_np, dev) if self.routes_stage_np is not None else None
    if self._dp_grad_desc_np is not None and len(self.ddesc_np):
      self._dp_grad_desc = up(self._dp_grad_desc_np, dev)
    self._refresh_tables()

  def _desc_hotness(self, descs) -> np.ndarray:
    """ids per sample of every descriptor (ragged inputs: their reserved capacity / 2)."""
    hot = descs["hotness"].astype(np.int64).copy()
    rag = hot == 0
    if rag.any():
      cap = max([abs(h) for h in self.hots if h < 0] + [2])
      hot[rag] = max(1, cap // 2)
    return hot

  @staticmethod
  def _tile_samples(descs, hot) -> int:
    if not len(descs):
      return 32
    avg = max(1, int(hot.mean()))
    if avg <= 4:
      return 32
    # never fewer samples than one warp instruction covers for the narrowest table
    lpr = 1
    while lpr < (int(descs["width"].min()) + 3) // 4 and lpr < 32:
      lpr *= 2
    return int(max(32 // lpr, min(32, 64 // avg), 1))

  def _refresh_tables(self):
    opt = self.de._fused_optimizer
    t = self.tdesc_np
    for m, layer in enumerate(self.mp_layers):
      t[m]["weight"] = self._ptr(_weight(layer))
      st = self.opt_state.get(m)
      c = self.caches.get(m)
      if c is not None:
        if [s.data_ptr() for s in c.host_state] != [s.data_ptr() for s in st or []]:
          c.invalidate()  # new host state (its old rows were flushed by reset_optimizer_state)
          c.set_state(st or [])
        t[m]["weight"] = c.weight.data_ptr()
        st = c.state
      t[m]["state0"] = self._ptr(st[0]) if st else 0
      t[m]["state1"] = self._ptr(st[1]) if st and len(st) > 1 else 0
    self.tdesc = _native.upload_struct_array(t, self.device) if len(t) else None
    self._tables_dirty = False
    # a trainer that shares its learning-rate word with the engine (DLRMTrainStep) owns it: a
    # refresh in the middle of its zero-lr graph warm-up must not switch the rate back on
    if opt is not None and not self._lr_external:
      self.lr_t.fill_(opt["lr"])

  # ------------------------------------------------------------------ optimizer state
  def reset_optimizer_state(self):
    self.flush_offload_cache(invalidate=True)
    self.opt_state = {}
    opt = self.de._fused_optimizer
    if opt is None:
      return
    kind = opt["kind"]
    self.step_t.fill_(float(opt.get("step", 0)))

    sdt = self.state_dtype

    def like(w, value, shape=None, dtype=torch.float32):
      # (a bf16 initial value is the round-to-nearest of ``value``)
      t = torch.full(shape or tuple(w.shape), value, dtype=dtype, device=w.device)
      # state of offloaded tables stays on the host (pinned, read zero-copy by the kernels)
      return t.pin_memory() if not (w.is_cuda or self.dry) else t

    for m, layer in enumerate(self.mp_layers):
      w = _weight(layer)
      if kind == "adagrad":
        self.opt_state[m] = [like(w, opt["initial_accumulator_value"], dtype=sdt)]
      elif kind == "rowwise_adagrad":
        self.opt_state[m] = [like(w, opt["initial_accumulator_value"], (w.shape[0],))]
      elif kind == "adam":
        self.opt_state[m] = [like(w, 0.0, dtype=sdt), like(w, 0.0, dtype=sdt)]
    self._tables_dirty = True

  @property
  def state_dtype(self) -> torch.dtype:
    """Storage of the element-wise optimizer state (Adagrad accumulator, Adam moments)."""
    opt = self.de._fused_optimizer
    return opt.get("state_dtype", torch.float32) if opt is not None else torch.float32

  def update_lr(self, lr: float):
    self.lr_t.fill_(lr)

  def share_lr(self, lr_t: torch.Tensor):
    """Use the caller's device-resident learning rate (one word, fp32) for the fused update:
    a trainer then changes the dense and the embedding rate with a single fill, and the engine
    never writes it."""
    self.lr_t = lr_t
    self._lr_external = True

  def step_count(self) -> int:
    """Optimizer steps applied so far (device counter: survives CUDA-graph replays)."""
    return int(round(float(self.step_t.item())))

  def optimizer_state_dict(self) -> Dict[str, Any]:
    """Local (sharding dependent) optimizer state; see
    :meth:`DistributedEmbedding.get_optimizer_state` for the global, resharding-safe layout."""
    return {"state": {m: [s.detach().cpu() for s in st] for m, st in self.opt_state.items()},
            "step": self.step_count()}

  def load_optimizer_state_dict(self, state):
    if not self.opt_state:
      self.reset_optimizer_state()
    for m, tensors in state.get("state", {}).items():
      for dst, src in zip(self.opt_state[int(m)], tensors):
        dst.copy_(src)
    step = int(state.get("step", 0))
    self.step_t.fill_(float(step))
    if self.de._fused_optimizer is not None:
      self.de._fused_optimizer["step"] = step

  # ------------------------------------------------------------------ forward
  def prepare(self, local_batch: int, hotness: Sequence[int], ids64: bool = False):
    """Allocate buffers up front (e.g. so a data loader can H2D-copy straight into
    ``input_views``); ``local_batch`` is the per-call batch of the inputs."""
    key = (int(local_batch), tuple(int(h) for h in hotness), bool(ids64))
    if key != self._key:
      self._build(*key)
    return self

  @property
  def input_views(self) -> List[torch.Tensor]:
    """``[batch, hotness]`` views of the staging buffer, one per input (dp_input mode)."""
    return self.in_views

  def _ragged_capacity(self, inputs, b: int) -> int:
    """Ids-per-sample capacity reserved for ragged inputs: user set
    (``DistributedEmbedding.ragged_capacity``) or 2x the largest mean hotness seen at build time,
    agreed on by all ranks (symmetric buffers must have one size)."""
    cap = getattr(self.de, "ragged_capacity", None)
    if cap is None:
      need = max(int(x.values.numel()) for x in inputs if isinstance(x, RaggedIds))
      cap = max(8, 2 * -(-need // max(b, 1)))
      if self.W > 1:
        t = torch.tensor([cap], dtype=torch.int64, device=self.device)
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX, group=self.de.group)
        cap = int(t.item())
      self.de.ragged_capacity = cap
    return int(cap)

  def stage(self, inputs):
    b = inputs[0].nrows if isinstance(inputs[0], RaggedIds) else int(inputs[0].shape[0])
    any_rag = any(isinstance(x, RaggedIds) for x in inputs)
    cap = self._ragged_capacity(inputs, b) if any_rag else 0
    hots = tuple(-cap if isinstance(x, RaggedIds) else (1 if x.dim() == 1 else int(x.shape[1]))
                 for x in inputs)
    ids64 = any((x.values if isinstance(x, RaggedIds) else x).dtype == torch.int64 for x in inputs)
    if self._key is None or self._key[0] != b or self._key[1] != hots or \
        (ids64 and not self._key[2]):
      self._build(b, hots, ids64)
    if self.de.dp_input:
      for i, (v, x) in enumerate(zip(self.in_views, inputs)):
        if isinstance(x, RaggedIds):
          n = int(x.values.numel())
          if n > v.numel():
            raise ValueError(
                f"ragged input {i} holds {n} ids but only {v.numel()} are reserved; raise "
                "DistributedEmbedding.ragged_capacity (ids per sample) on every rank")
          v.view(-1)[:n].copy_(x.values, non_blocking=True)
          self.split_views[i].copy_(x.row_splits, non_blocking=True)
        elif x.data_ptr() != v.data_ptr():
          v.copy_(x.reshape(v.shape), non_blocking=True)
    else:
      for li, x in enumerate(inputs):
        pos = self.col_items[li]
        if isinstance(x, RaggedIds):
          n = int(x.values.numel())
          if n > self.B * cap:
            raise ValueError(f"ragged input {li} holds {n} ids, capacity is {self.B * cap}")
          self.ids_mp[pos:pos + n].copy_(x.values, non_blocking=True)
          j = self.my_ragged_mp.index(li)
          self.goff[j * (self.B + 1):(j + 1) * (self.B + 1)].copy_(x.row_splits,
                                                                     non_blocking=True)
        else:
          n = x.numel()
          self.ids_mp[pos:pos + n].copy_(x.reshape(-1), non_blocking=True)

  def forward(self, inputs, concat: bool):
    self.stage(inputs)
    return self.run(concat)

  def run(self, concat: bool = True):
    """Forward on already staged inputs (see :meth:`prepare` / :attr:`input_views`)."""
    if self.de._fused_optimizer is not None and not self.opt_state and \
        self.de._fused_optimizer["kind"] != "sgd":
      self.reset_optimizer_state()
    if self._tables_dirty:
      self._refresh_tables()
    weights = [_weight(l) for l in list(self.de.dp_layers) + self.mp_layers]
    # a forward that records a backward is a training pass: the cache marks its rows dirty
    train = torch.is_grad_enabled() and any(w.requires_grad for w in weights)
    out = _FusedFn.apply(self, self._token, train, *weights)
    if concat:
      return out
    return list(torch.split(out, self.out_widths, dim=1))

  def _run_forward(self, train: bool = True):
    with nvtx.range("emb_forward"):
      self.launch_forward(train)
      self.wait_output()
      return self.out

  @property
  def has_mp(self) -> bool:
    return self.fwd_main is not None or self.fwd_rs is not None

  @property
  def out_needs_reduce(self) -> bool:
    """Multi-hot row-sliced inputs: the requester still has to sum the owners' partial pools
    (``wait_output`` does it); a fused consumer can only fold the wait when this is False."""
    return self.rs_buf is not None

  def launch_forward(self, train: bool = True):
    """Index exchange + lookups.  ``train``: the step updates the tables after this forward (the
    offload cache then marks the rows it serves dirty); False for a forward-only pass.  The pooled rows of this rank's tables are on their way to the
    requesters when this returns; the *consumer* of ``self.out`` must wait for the owners'
    "output ready" signals (:meth:`wait_output`, or ``sync_out_wait()`` folded into its kernel)."""
    ops, W, rank = self.ops, self.W, self.rank
    B, lb = self.B, self.lb
    wait_ids = -1
    if W > 1 and self.has_mp:
      if self.id_mode == "push":
        # head: every owner has consumed last step's ids; tail: my ids are in the owners' buffers
        ops.push_segments(self.push_segs, self.in_flat, self.ids_ptrs, self.max_push,
                          self._sync(wait_abs=CH_CONSUMED, signal=CH_IDS))
        wait_ids = CH_IDS
      elif self.id_mode == "pull":
        self.ctx.barrier(CH_BARRIER0)  # every rank's ids are staged
        if self.segs is not None:
          ops.gather_segments(self.segs, self.in_ptrs, self.ids_mp, self.max_seg)
        if self.rsegs is not None:
          ops.gather_ragged(self.rsegs, self.in_ptrs, self.split_ptrs, self.ids_mp, self.goff,
                            self.lb, self.max_rcap)
      else:  # model-parallel inputs: nothing to exchange, but the output buffers of the
        # requesters may only be overwritten once they are done with the previous step
        ops.sync_only(self._sync(signal=CH_IDS))
        wait_ids = CH_IDS
    if self._cache_plan:
      # the cache pass reads the arrived ids: it takes the "ids ready" wait, the lookups then
      # run without one.  Its write-back of last step's rows is ordered behind last step's
      # update by stream order (see DESIGN.md, offload cache)
      if wait_ids >= 0:
        ops.sync_only(self._sync(wait=wait_ids))
        wait_ids = -1
      self._run_cache_pass(train)
    if self.ddesc is not None:
      ops.lookup_fwd(self.ddesc, len(self.ddesc_np), lb, lb, lb, self.out_stride, [],
                     [self.out.data_ptr()], 0, self.ids64, self.act, self.vec4, [],
                     self._tile_samples(self.ddesc_np, self._desc_hotness(self.ddesc_np)))
    for k, (descs, n, tile) in enumerate(self.fwd_launches):
      last = k == len(self.fwd_launches) - 1 and self.fwd_rs is None
      ops.lookup_fwd(descs, n, B, B, lb, self.out_stride, [], self.out_ptrs, rank, self.ids64,
                     self.act, self.vec4,
                     self._sync(wait=wait_ids, signal=CH_OUT if last else -1), tile, self.tab,
                     self.fwd_vec8)
      wait_ids = -1  # later launches of this stream are ordered behind the wait
    if self.fwd_rs is not None:
      ops.lookup_fwd(self.fwd_rs, len(self.fwd_rs_np), B, B, lb, self.rs_width, [], self.rs_ptrs,
                     rank, self.ids64, 0, self.vec4, self._sync(wait=wait_ids, signal=CH_OUT),
                     self.fwd_rs_tile, self.tab, self.fwd_vec8)

  def sync_out_wait(self):
    """``sync`` spec that makes a consumer kernel wait for the owners' "output ready" signals."""
    return self._sync(wait=CH_OUT) if (self.W > 1 and self.has_mp) else []

  def wait_output(self):
    """Consumer side of the forward: wait until every owner's rows have landed in ``self.out``
    and sum the partial pools of multi-hot row-sliced inputs."""
    if self.W > 1 and self.has_mp:
      self.ops.sync_only(self._sync(wait=CH_OUT))
    if self.rs_buf is not None:
      self.ops.rowslice_reduce(self.rs, self.out.data_ptr(), self.out_stride, self.act,
                               self.rs_cols_t)

  # ------------------------------------------------------------------ backward
  def _run_backward(self, grad_out: torch.Tensor):
    ops, de = self.ops, self.de
    lb = self.lb
    if grad_out.dtype not in DTYPE_CODE or grad_out.stride(-1) != 1:
      grad_out = grad_out.float().contiguous()
    self._grad_out_live = grad_out if self.dry else None  # addressable for the plan interpreter
    # gradient all-to-all: every piece of my rows goes straight into its owner's receive buffer
    if self.routes_mp is not None:
      ops.push_grad(self.routes_mp, len(self.routes_mp_np), grad_out, self.act, 1.0,
                    self._sync(signal=CH_GRAD))
    grads: List[Optional[torch.Tensor]] = []
    # replicated tables: dense local gradients (all-reduced later with the MLP gradients), read
    # straight from the incoming gradient; persistent buffers + descriptors, one launch
    if len(de.dp_layers):
      need = [_weight(l).requires_grad for l in de.dp_layers]
      if any(need) and self._dp_grad_desc is not None:
        self._dp_grad_flat.zero_()
        ops.scatter_add_bwd(self._dp_grad_desc, len(self.ddesc_np), lb, lb, lb,
                            grad_out.stride(0), [], [grad_out.data_ptr()], 0, 1.0, 0, self.ids64,
                            DTYPE_CODE[grad_out.dtype], self._grad_vec4(grad_out), False, [],
                            False)
      for m in range(len(de.dp_layers)):
        grads.append(self._dp_grad_views[m].clone() if need[m] else None)
    grads += self._backward_mp()
    return grads

  def _grad_vec4(self, g: torch.Tensor) -> bool:
    return self.vec4 and g.stride(0) % 4 == 0 and g.data_ptr() % 16 == 0

  def set_dp_grad_targets(self, targets: Optional[Sequence[torch.Tensor]]):
    """Persistent dense-gradient buffers of the replicated tables, one fp32 ``[rows, width]``
    tensor per ``de.dp_layers`` entry (e.g. slices of a flat all-reduce bucket).  The caller
    zeroes them every step; :meth:`backward_inplace` accumulates the local-batch gradient into
    them, so a hand-scheduled step can all-reduce and apply them with its dense parameters."""
    if targets is not None:
      targets = list(targets)
      if len(targets) != len(self.de.dp_layers):
        raise ValueError(f"expected {len(self.de.dp_layers)} targets, got {len(targets)}")
      for t, layer in zip(targets, self.de.dp_layers):
        w = _weight(layer)
        if t.dtype != torch.float32 or tuple(t.shape) != tuple(w.shape) or not t.is_contiguous():
          raise ValueError("dp gradient targets must be contiguous fp32 tensors of the table shape")
    self._dp_targets = targets
    self._dp_target_desc = None

  def _scatter_dp_grads(self):
    """Local-batch gradient of every replicated table into its persistent target (one launch);
    the gradient rows come from ``self.grad`` (requester layout, written by a fused producer)."""
    if not len(self.ddesc_np):
      return
    key = (self._key, tuple(t.data_ptr() for t in self._dp_targets))
    if self._dp_target_desc is None or self._dp_target_desc[0] != key:
      d = self.ddesc_np.copy()
      for j in range(len(d)):
        d[j]["table"] = self._dp_targets[int(d[j]["local_table"])].data_ptr()
      self._dp_target_desc = (key, _native.upload_struct_array(d, self.device), len(d))
    _, dd, n = self._dp_target_desc
    self.ops.scatter_add_bwd(dd, n, self.lb, self.lb, self.lb, self.total_width, [],
                             [self.grad.data_ptr()], 0, 1.0, 0, self.ids64, self.act, self.vec4,
                             False, [], self.staged_dp)

  @property
  def streamed_push(self) -> bool:
    return self.gstage is not None

  def launch_streamed_push(self, blocks: int = 32):
    """The copy kernel of the streamed gradient push (see :meth:`enable_streamed_push`): launch
    it on its own stream right *after* the producer (it spins on the producer's progress, so it
    must never sit in front of it in a hardware queue the two streams share); the producer gets
    ``routes_stage``, ``push_counters`` (zeroed by the caller beforehand) and
    ``push_chunk_rows``."""
    src, dst, row_bytes = self.push_plan
    self.ops.stream_push(src, dst, row_bytes, self.push_counters, self.push_chunk_rows, self.lb,
                         blocks, self._sync(signal=CH_GRAD))

  def sync_grad_signal(self):
    """``sync`` spec for a fused gradient producer (it stores through ``routes_all`` and
    signals "gradient ready" from its tail)."""
    return self._sync(signal=CH_GRAD) if (self.W > 1 and self.mpdesc is not None) else []

  def backward_inplace(self, producer: Optional["ProducerUpdate"] = None):
    """Backward when a fused producer (e.g. the DLRM interaction backward) already pushed the
    gradient through ``routes_all`` and signalled: fused table update; replicated tables
    accumulate their dense gradient into the targets given to :meth:`set_dp_grad_targets`.
    ``producer``: the :meth:`producer_update` whose tables the producer updated itself; only the
    remaining tables are scattered."""
    if len(self.de.dp_layers):
      if getattr(self, "_dp_targets", None) is None:
        raise RuntimeError("backward_inplace needs set_dp_grad_targets() for replicated tables")
      self._scatter_dp_grads()
    self._backward_mp(producer)

  def _atomic_sgd(self) -> bool:
    """The SGD update is one atomic scatter of the gradient rows into the tables.  Not with
    weight decay: the scatter adds each id's gradient on its own, so with duplicate ids it could
    not apply the decay exactly once per row; SGD with decay takes the sorted update."""
    opt = self.de._fused_optimizer
    return opt is not None and opt["kind"] == "sgd" and not opt.get("deterministic", False) and \
        opt.get("weight_decay", 0.0) == 0.0 and not self.has_offload and self.tab == 0

  def producer_update(self, dim: int, min_rows: int) -> Optional["ProducerUpdate"]:
    """The SGD table update a single-GPU gradient producer can apply itself.

    The producer (the DLRM interaction backward) holds every sample's finished gradient row of
    feature ``f`` in columns ``[f * dim, (f + 1) * dim)`` of ``out``.  Reducing it straight into
    the table row saves the write of the row into the receive buffer and the scatter's read of
    it.  Tables with fewer than ``min_rows`` rows stay with the staged scatter, which sums the
    samples of a 32-sample tile that hit the same row before it reduces them.

    Returns a :class:`ProducerUpdate` (``interact_args()`` for ``ops.interact_bwd``; pass it to
    :meth:`backward_inplace`), or None when the step does not qualify: one rank, the atomic SGD
    update, one-hot 128-wide inputs of a single ``dim``-wide output row each, and at least one
    table of ``min_rows`` rows or more."""
    if self._key is None or self.W != 1 or not self._atomic_sgd() or not self.vec4 or \
        self.any_ragged or dim != 128 or self.mpdesc is None or \
        not any(_weight(l).requires_grad for l in self.mp_layers):
      return None
    cache = getattr(self, "_producer_split", None)
    if cache is None or cache[0] != (self._key, dim, min_rows) or cache[1] is not self.mpdesc:
      n_feat = len(self.out_cols) - 1
      apply = np.zeros(n_feat, dtype=INPUT_DESC)
      taken = np.zeros(self.n_mp_inputs, dtype=bool)
      if self.out_cols == [dim * f for f in range(n_feat + 1)] and n_feat <= 31:
        for i, d in enumerate(self.cdesc_np):
          f, off = divmod(int(d["dst_col"]), dim)
          if off == 0 and int(d["width"]) == dim and int(d["hotness"]) == 1 and \
              int(d["offsets"]) == 0 and int(d["ids"]) != 0 and int(d["sub_rows"]) >= min_rows:
            apply[f] = d
            taken[i] = True
      rest = self.mpdesc_np[~taken]
      rest_dev = _native.upload_struct_array(rest, self.device) if len(rest) else None
      apply_t = torch.from_numpy(apply.view(np.uint8).copy()) if taken.any() else None
      self._producer_split = ((self._key, dim, min_rows), self.mpdesc, apply_t, rest_dev, len(rest))
    _, mpdesc, apply_t, rest_dev, n_rest = self._producer_split
    if apply_t is None:
      return None
    gscale = 0.0 if self._dry_updates else self.de.mp_grad_scale
    return ProducerUpdate(mpdesc, apply_t, -gscale, self.lr_t.data_ptr(), self.ids64, rest_dev,
                          n_rest)

  def _backward_mp(self, producer: Optional["ProducerUpdate"] = None
                   ) -> List[Optional[torch.Tensor]]:
    with nvtx.range("emb_backward_update"):
      return self._backward_mp_impl(producer)

  def _backward_mp_impl(self, producer: Optional["ProducerUpdate"] = None
                        ) -> List[Optional[torch.Tensor]]:
    ops, de = self.ops, self.de
    if producer is not None and (producer.mpdesc is not self.mpdesc or not self._atomic_sgd()):
      raise ValueError("the producer update was built for another plan or optimizer: call "
                       "producer_update() for the current one")
    n_mp = len(self.mp_layers)
    if self.mpdesc is None:
      return [None] * n_mp
    multi = self.W > 1
    if not any(_weight(l).requires_grad for l in self.mp_layers):
      if multi:  # keep the signalling protocol in step: consume the gradient signal
        ops.sync_only(self._sync(wait=CH_GRAD, signal=CH_CONSUMED))
      return [None] * n_mp
    opt = de._fused_optimizer
    if opt is None and self.caches:
      raise RuntimeError("the offload cache updates its rows with the fused optimizer: call "
                         "DistributedEmbedding.set_optimizer() before training a cached model")
    if opt is not None and opt["kind"] != "sgd" and not self.opt_state:
      self.reset_optimizer_state()
    if self._tables_dirty:
      self._refresh_tables()
    B = self.B
    gscale = 0.0 if self._dry_updates else de.mp_grad_scale
    # 16-bit tables always take the sorted, deduplicated update, SGD included: each row then has
    # exactly one writer per step and is stochastically rounded once.  An atomic 16-bit add would
    # round to nearest on every duplicate id (dropping sub-half-ulp updates) and its result
    # would depend on the order of the adds.
    if self._atomic_sgd():
      descs, n = self.mpdesc, self.n_mp_inputs
      if producer is not None:  # the producer updated the large tables itself
        descs, n = producer.rest_descs, producer.n_rest
        if n == 0:
          return [None] * n_mp
      # head: every requester's gradient rows have landed; tail: ids + gradients are consumed
      ops.scatter_add_bwd(descs, n, B, B, B, self.recv_width, [],
                          self.recv_ptr, 0, -gscale, self.lr_t.data_ptr(), self.ids64,
                          self.act, self.vec4, self.vec8,
                          self._sync(wait=CH_GRAD, signal=CH_CONSUMED), self.staged_update)
      return [None] * n_mp
    if multi:
      ops.sync_only(self._sync(wait=CH_GRAD))
    keys, items, seg, n_unique = ops.sort_items(self.mpdesc, self.tdesc, n_mp, self.n_mp_inputs,
                                                B, B, [], self.ids64, self.n_items,
                                                self.total_rows, self.any_ragged)
    if opt is not None:
      if not self._dry_updates:
        self.step_t.add_(1.0)  # device counter: bias corrections stay right under graph replay
      kind = _OPT_KIND[opt["kind"]]
      if self._dry_updates and opt["kind"] == "adam":
        kind = _OPT_KIND["sgd"]  # a zero gradient would still decay Adam's moments
      # a dry update has no decay either: weight_decay * w would move the weights and feed the
      # Adagrad accumulators on every warm-up pass
      wd = 0.0 if self._dry_updates else opt["weight_decay"]
      ops.segment_update(self.mpdesc, self.tdesc, n_mp, B, B, self.recv_width, self.recv_ptr,
                         keys, items, seg, n_unique, kind, opt["lr"],
                         opt["eps"], opt["beta1"], opt["beta2"], 1.0, 1.0, gscale,
                         wd, self.lr_t.data_ptr(), None, None, self.max_width,
                         self.act, self.vec4, self._balanced_scratch(), self.step_t.data_ptr(),
                         self.tab, DTYPE_CODE[self.state_dtype])
      if multi:
        ops.sync_only(self._sync(signal=CH_CONSUMED))
      return [None] * n_mp
    # no fused optimizer: materialise deduplicated sparse gradients (reference semantics)
    emit_keys = torch.empty(self.n_items, dtype=torch.int64, device=self.device)
    emit_rows = torch.empty(self.n_items, self.max_width, dtype=torch.float32, device=self.device)
    ops.segment_update(self.mpdesc, self.tdesc, n_mp, B, B, self.recv_width, self.recv_ptr, keys,
                       items, seg, n_unique, _native.OPT_EMIT, 0.0, 0.0, 0.0, 0.0, 1.0, 1.0,
                       de.mp_grad_scale, 0.0, 0, emit_keys, emit_rows, self.max_width, self.act,
                       self.vec4, None, 0)
    if multi:
      ops.sync_only(self._sync(signal=CH_CONSUMED))
    nu = int(n_unique.item())
    emit_keys, emit_rows = emit_keys[:nu], emit_rows[:nu]
    bases = [int(x) for x in self.tdesc_np["key_base"]] + [self.total_rows]
    bounds = torch.searchsorted(emit_keys, torch.tensor(bases, device=self.device)).tolist()
    out = []
    for m, layer in enumerate(self.mp_layers):
      w = _weight(layer)
      lo, hi = bounds[m], bounds[m + 1]
      ids = (emit_keys[lo:hi] - bases[m]).unsqueeze(0).to(w.device)
      # a fresh [nnz, width] buffer with canonical strides: for nnz == 1 ``.contiguous()`` is a
      # no-op on the padded view (row stride max_width) and PyTorch's sparse -> dense kernels
      # then address the destination with that stride (heap overflow found by the plan fuzzer)
      # (in the table's dtype: autograd hands a parameter gradients of its own dtype)
      rows = torch.empty(hi - lo, w.shape[1], dtype=w.dtype, device=emit_rows.device)
      rows.copy_(emit_rows[lo:hi, :w.shape[1]])
      rows = rows.to(w.device)
      out.append(torch.sparse_coo_tensor(ids, rows, size=tuple(w.shape), is_coalesced=True,
                                         check_invariants=False))
    return out

  def _balanced_scratch(self):
    """Zero-initialised scratch rows of the occurrence-balanced update (kept zero by the
    kernels); None selects the per-unique-row kernel (wide tables)."""
    if not self.vec4 or self.max_width > 128 or self.n_items == 0:
      return None
    sw = (self.max_width + 3) // 4 * 4
    need = ((self.n_items + 31) // 32) * sw
    cur = getattr(self, "_scratch", None)
    if cur is None or cur.numel() < need:
      self._scratch = torch.zeros(need, dtype=torch.float32, device=self.device)
    return self._scratch

"""Communication runtime: one process per GPU, ``torch.distributed`` for bootstrap and cold
paths, peer-mapped *symmetric buffers* (cudaMalloc + CUDA IPC) for the hot paths.

Every rank allocates the same set of buffers; handles are exchanged once through the process
group and opened with ``cudaIpcOpenMemHandle`` so each rank holds a device pointer to every
peer's copy.  Kernels then load/store peer HBM directly over NVLink 4 / NVSwitch.  Cross-rank
ordering uses a signal pad of per-(channel, writer) epoch words written with ``st.release.sys``
and polled with ``ld.acquire.sys`` under a bounded-spin watchdog (no infinite device spins).

Replaces the Horovod layer of the reference (SURVEY.md section 5.8; dist_model_parallel.py:22-24).
"""
from __future__ import annotations

import os
import socket
from typing import Dict, List, Optional

import torch
import torch.distributed as dist

from ..ops import _native

# Cycles a device-side flag wait may spin before the watchdog records the missing peer in
# host-mapped memory and traps the kernel (~60 s at 2 GHz; 0 = wait forever).  A timeout is
# fatal by design: continuing past a lost peer would consume stale ids / gradients and corrupt
# the tables silently, whereas a trapped kernel surfaces as a CUDA error on every later call.
DEFAULT_TIMEOUT_CYCLES = int(os.environ.get("DE_B200_FLAG_TIMEOUT_CYCLES", str(120_000_000_000)))
NUM_CHANNELS = 16
# signalling channels of the fused embedding engine (kernels wait / signal on them, see
# ops/csrc/common.cuh sync_head / sync_tail); legacy two-way barriers use 8..10, the dense
# all-reduce 14..15
CH_IDS, CH_OUT, CH_GRAD, CH_CONSUMED = 0, 1, 2, 3
CH_BARRIER0 = 8


def dist_ready() -> bool:
  return dist.is_available() and dist.is_initialized()


def host_identity() -> str:
  """Identifies the OS instance a rank runs on (CUDA IPC handles only open inside one)."""
  boot = ""
  try:
    with open("/proc/sys/kernel/random/boot_id", encoding="ascii") as f:
      boot = f.read().strip()
  except OSError:
    pass
  return f"{socket.gethostname()}/{boot}"


def single_p2p_domain(identities: List[str], max_peers: int) -> bool:
  """True when all ranks can map each other's memory: one host, at most ``max_peers`` ranks."""
  return len(identities) <= max_peers and len(set(identities)) == 1


class SymmetricBuffer:
  """A same-sized device buffer on every rank, with peer pointers to all copies."""

  def __init__(self, ctx: "CommContext", nbytes: int, name: str = ""):
    self.ctx = ctx
    self.name = name
    self.nbytes = int(nbytes)
    dev = ctx.device
    ops = _native.require()
    self.local = ops.symm_alloc(self.nbytes, dev.index)  # uint8 tensor, zero filled
    self.ptrs: List[int] = [0] * ctx.world_size
    self._opened: List[int] = []
    self.ptrs[ctx.rank] = self.local.data_ptr()
    if ctx.world_size > 1:
      handle = ops.ipc_get_handle(self.local)
      gathered: List[Optional[torch.Tensor]] = [None] * ctx.world_size
      dist.all_gather_object(gathered, handle.numpy().tobytes(), group=ctx.group)
      for r, raw in enumerate(gathered):
        if r == ctx.rank:
          continue
        h = torch.frombuffer(bytearray(raw), dtype=torch.uint8)
        p = ops.ipc_open(h, dev.index)
        self.ptrs[r] = p
        self._opened.append(p)

  def view(self, dtype: torch.dtype, shape, byte_offset: int = 0) -> torch.Tensor:
    """Typed view of the local copy."""
    n = 1
    for s in shape:
      n *= int(s)
    nbytes = n * torch.empty((), dtype=dtype).element_size()
    assert byte_offset + nbytes <= self.local.numel(), (self.name, byte_offset, nbytes,
                                                         self.local.numel())
    return self.local[byte_offset:byte_offset + nbytes].view(dtype).view(*shape)

  def peer_ptrs(self, byte_offset: int = 0) -> List[int]:
    return [p + byte_offset for p in self.ptrs]

  def close(self):
    if self._opened:
      ops = _native.require()
      for p in self._opened:
        ops.ipc_close(p, self.ctx.device.index)
      self._opened = []

  def __del__(self):
    try:
      self.close()
    except Exception:  # pylint: disable=broad-except
      pass


class MulticastBuffer:
  """Symmetric buffer that additionally has an NVSwitch *multicast* mapping (NVLS): one
  ``multimem.ld_reduce`` returns the sum over all GPUs computed inside the switch and one
  ``multimem.st`` broadcasts to all of them.  Allocation and handle exchange go through
  ``torch.distributed._symmetric_memory`` (CUDA VMM + fabric/fd handles); the kernels are ours.
  Same surface as :class:`SymmetricBuffer` plus ``mc_ptr``."""

  def __init__(self, ctx: "CommContext", nbytes: int, name: str = ""):
    import torch.distributed._symmetric_memory as symm_mem  # pylint: disable=import-outside-toplevel
    self.ctx, self.name = ctx, name
    self.nbytes = (int(nbytes) + 255) // 256 * 256
    group = ctx.group if ctx.group is not None else dist.group.WORLD
    with torch.cuda.device(ctx.device):
      self.local = symm_mem.empty(self.nbytes, dtype=torch.uint8, device=ctx.device)
      self.local.zero_()
      self._hdl = symm_mem.rendezvous(self.local, group)
    self.ptrs = [int(p) for p in self._hdl.buffer_ptrs]
    self.mc_ptr = int(self._hdl.multicast_ptr) if self._hdl.has_multicast_support else 0
    if self.mc_ptr == 0:
      raise RuntimeError("no multicast support")
    torch.cuda.synchronize(ctx.device)

  view = SymmetricBuffer.view
  peer_ptrs = SymmetricBuffer.peer_ptrs

  def close(self):
    pass


class CommContext:
  """Rank / world bookkeeping plus the device-side synchronisation state of one process group."""

  _default: Optional["CommContext"] = None

  def __init__(self, group=None, device: Optional[torch.device] = None):
    if dist_ready():
      self.group = group
      self.rank = dist.get_rank(group)
      self.world_size = dist.get_world_size(group)
    else:
      self.group = None
      self.rank, self.world_size = 0, 1
    if device is None:
      if torch.cuda.is_available():
        device = torch.device("cuda", torch.cuda.current_device())
      else:
        device = torch.device("cpu")
    self.device = torch.device(device)
    self.is_cuda = self.device.type == "cuda"
    self.p2p = False
    self.signal: Optional[SymmetricBuffer] = None
    self._epochs: Dict[int, torch.Tensor] = {}
    self.error_flag: Optional[torch.Tensor] = None
    self.error_ptr = 0
    self.sync_state: Optional[torch.Tensor] = None
    self.sync_handle = -1
    self.timeout_cycles = DEFAULT_TIMEOUT_CYCLES
    # Peer mappings need every rank on one host with peer access; otherwise (multi-node jobs,
    # PCIe boxes without P2P) the context stays usable for bookkeeping and callers fall back to
    # torch.distributed collectives (DistributedEmbedding backend "torch", NCCL all-reduce).
    self.p2p_unavailable_reason: Optional[str] = None
    if self.is_cuda and _native.available():
      reason = self._p2p_obstacle()
      if reason is None:
        self._init_p2p()
      else:
        self.p2p_unavailable_reason = reason

  # -- construction helpers ---------------------------------------------------------------
  @classmethod
  def default(cls, device=None) -> "CommContext":
    if cls._default is None or (device is not None and
                                torch.device(device) != cls._default.device) or (
                                    cls._default.world_size != (dist.get_world_size()
                                                                if dist_ready() else 1)):
      cls._default = CommContext(device=device)
    return cls._default

  _by_group: Dict[int, "CommContext"] = {}

  @classmethod
  def for_group(cls, group, device=None) -> "CommContext":
    """Context of a process (sub)group; ``None`` is the default (world) group.  Collective: all
    members of the group must call it at the same point."""
    if group is None:
      return cls.default(device)
    ctx = cls._by_group.get(id(group))
    if ctx is None or (device is not None and torch.device(device) != ctx.device):
      ctx = CommContext(group=group, device=device)
      cls._by_group[id(group)] = ctx
    return ctx

  def _p2p_obstacle(self) -> Optional[str]:
    """None when symmetric peer mappings can be set up; else why not (same answer on all ranks)."""
    if self.world_size == 1:
      return None
    ids = [None] * self.world_size
    peer_ok = True
    me = self.device.index if self.device.index is not None else torch.cuda.current_device()
    for d in range(torch.cuda.device_count()):
      if d != me and not torch.cuda.can_device_access_peer(me, d):
        peer_ok = False
    with torch.cuda.device(self.device):  # NCCL object collectives stage through this device
      dist.all_gather_object(ids, (host_identity(), peer_ok), group=self.group)
    if not single_p2p_domain([i[0] for i in ids], _native.MAX_PEERS):
      return (f"{self.world_size} ranks on {len({i[0] for i in ids})} host(s); peer mappings need "
              f"one host and at most {_native.MAX_PEERS} ranks")
    if not all(i[1] for i in ids):
      return "CUDA peer access is not available between all GPUs of this host"
    return None

  def _init_p2p(self):
    with torch.cuda.device(self.device):
      ops = _native.require()
      self.signal = SymmetricBuffer(self, NUM_CHANNELS * _native.MAX_PEERS * 4, "signal_pad")
      # watchdog word in pinned host memory: still readable after a kernel trapped
      self.error_flag = torch.zeros(1, dtype=torch.int32).pin_memory()
      self.error_ptr = int(ops.host_device_pointer(self.error_flag))
      # wait / signal epochs + block counters of the signalling protocol (device resident)
      self.sync_state = torch.zeros(_native.SYNC_STATE_WORDS, dtype=torch.int32,
                                    device=self.device)
      self.sync_handle = int(ops.sync_ctx_create(self.signal.ptrs, self.sync_state, self.rank,
                                                 self.world_size, self.timeout_cycles,
                                                 self.error_ptr))
      if self.world_size > 1:
        dist.barrier(group=self.group)
      self.p2p = True

  def sync(self, wait: int = -1, wait_abs: int = -1, signal: int = -1, slot: Optional[int] = None):
    """Signalling spec for a native op (``int[] sync``): the kernel waits at its head for every
    peer's signal on channel ``wait`` (and/or until the peers have caught up with this rank's own
    signals on ``wait_abs``) and publishes ``signal`` to every peer from its tail.  Empty list
    on a single rank."""
    if self.world_size == 1 or not self.p2p:
      return []
    if slot is None:
      slot = signal if signal >= 0 else NUM_CHANNELS + max(wait, wait_abs, 0)
    return [self.sync_handle, int(wait), int(wait_abs), int(signal), int(slot)]

  def epoch(self, channel: int) -> torch.Tensor:
    """Device-resident epoch words of a channel ([0] epoch, [1] block counter): kernels bump them
    on the device so a captured CUDA graph can be replayed without host patching."""
    if channel not in self._epochs:
      self._epochs[channel] = torch.zeros(2, dtype=torch.int32, device=self.device)
    return self._epochs[channel]

  # -- collectives --------------------------------------------------------------------------
  def alloc(self, nbytes: int, name: str = "") -> SymmetricBuffer:
    if not self.p2p:
      raise RuntimeError("symmetric buffers need CUDA + the native extension" +
                         (f" ({self.p2p_unavailable_reason})" if self.p2p_unavailable_reason else ""))
    with torch.cuda.device(self.device):
      return SymmetricBuffer(self, nbytes, name)

  def alloc_multicast(self, nbytes: int, name: str = "") -> Optional[MulticastBuffer]:
    """Symmetric buffer with an NVSwitch multicast mapping, or None when NVLS is unavailable
    (single GPU, no NVSwitch, or the handle exchange is not permitted in this container)."""
    # opt-in (DE_B200_NVLS=1): it needs an NVSwitch system, and the P2P path needs nothing beyond
    # CUDA IPC
    if not self.p2p or self.world_size == 1 or os.environ.get("DE_B200_NVLS", "0") != "1":
      return None
    ok = 1
    buf = None
    try:
      buf = MulticastBuffer(self, nbytes, name)
    except Exception:  # pylint: disable=broad-except
      ok = 0
    # all ranks must take the same path
    flag = torch.tensor([ok], dtype=torch.int32, device=self.device)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.group)
    return buf if int(flag.item()) == 1 else None

  def barrier(self, channel: int = 0):
    """Device-side barrier on the current stream (no host synchronisation)."""
    if self.world_size == 1:
      return
    if not self.p2p:
      dist.barrier(group=self.group)
      return
    _native.ops().barrier(self.signal.ptrs, self.epoch(channel), self.rank, self.world_size,
                          channel, self.timeout_cycles, self.error_ptr)

  def allreduce_(self, buf: SymmetricBuffer, n_elems: int, dtype: torch.dtype, scale: float = 1.0,
                 channel: int = 15, byte_offset: int = 0, mc_ptr: int = 0, max_blocks: int = 0):
    """In-place sum (x scale) over all ranks of a symmetric buffer; one kernel, no NCCL.
    ``max_blocks`` > 0 caps the grid (use it when the all-reduce overlaps other kernels)."""
    if self.world_size == 1:
      if scale != 1.0:
        buf.view(dtype, (n_elems,), byte_offset).mul_(scale)
      return
    if mc_ptr == 0:
      mc_ptr = getattr(buf, "mc_ptr", 0)
      if mc_ptr:
        mc_ptr += byte_offset
    _native.ops().allreduce(buf.peer_ptrs(byte_offset), self.signal.ptrs, self.epoch(channel),
                            self.rank, self.world_size, n_elems, float(scale),
                            dtype == torch.bfloat16, channel, self.timeout_cycles, self.error_ptr,
                            mc_ptr, int(max_blocks))

  def check_errors(self):
    """Host check of the watchdog word (pinned host memory: no device synchronisation, and still
    readable after a timed-out kernel trapped the context)."""
    if self.error_flag is not None:
      v = int(self.error_flag[0])
      if v != 0:
        raise RuntimeError(
            f"rank {self.rank}: peer flag wait timed out waiting for rank {v - 1} - a rank is "
            "hung, crashed, or running a mismatched plan")

  # -- cold-path helpers (torch.distributed) ------------------------------------------------
  def all_gather_object(self, obj):
    if self.world_size == 1:
      return [obj]
    out = [None] * self.world_size
    dist.all_gather_object(out, obj, group=self.group)
    return out

  def broadcast_(self, tensor: torch.Tensor, src: int = 0):
    if self.world_size > 1:
      dist.broadcast(tensor, src=src, group=self.group)
    return tensor

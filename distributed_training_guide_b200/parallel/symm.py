"""NVLink symmetric memory: buffers every rank of a group can address directly.

This is the substrate the reference does not have (it only ever calls NCCL, SURVEY.md §5.8):
each rank ``cudaMalloc``s the same size outside the caching allocator, exports a CUDA-IPC handle,
handles are exchanged once through ``torch.distributed`` (NCCL/gloo is used for this bootstrap
only), and every rank maps its peers' buffers.  Collective *kernels* (``csrc/comm.cu``,
``csrc/fused_tp.cu``) then load/store peer memory over NVLink / NVSwitch and synchronise with
device-side epoch flags in a symmetric signal pad — no host round trips, no NCCL on the hot path.

``SymmGroup`` also runs on a single rank (N = 1: same kernels, no peers), which is how the
single-GPU chapter shares the fused optimizer path.
"""
from __future__ import annotations

import os
from typing import List, Optional

import torch
import torch.distributed as dist

from .. import _ext

_LIVE_GROUPS = []


def allocated_bytes() -> int:
    c = _ext.load(False)
    n = int(c.symm_allocated_bytes()) if c is not None and hasattr(c, "symm_allocated_bytes") else 0  # cudaMalloc'ed
    return n + sum(ch.size for g in _LIVE_GROUPS for ch in g._chunks if isinstance(ch, _VmmChunk))


def post_mortem(timeout_s: float = 5.0):
    """Signal-pad state of every live group, read on a side stream with a bounded wait so it also works while a
    kernel of this process is spinning on the device (a hung run's last words; used by bench.py's watchdog)."""
    lines = []
    for i, g in enumerate(list(_LIVE_GROUPS)):
        try:
            lines.append(f"symm group {i} (rank {g.rank}/{g.world}): " + g.describe_pads(timeout_s=timeout_s))
        except Exception as e:  # pragma: no cover - diagnostics only
            lines.append(f"symm group {i}: unavailable ({e!r})")
    return lines


class SymmBuffer:
    """One symmetric allocation: ``local`` (this rank's memory as a tensor) + every rank's base pointer
    (+ the NVSwitch multicast address of the allocation when it was bound to one, else 0)."""

    def __init__(self, local: torch.Tensor, ptrs: List[int], raw: torch.Tensor, mc_ptr: int = 0, handle=None):
        self.local = local
        self.ptrs = ptrs
        self._raw = raw  # keeps the allocation alive
        self.mc_ptr = int(mc_ptr or 0)
        self._handle = handle

    def elem_offset_of(self, view: torch.Tensor) -> int:
        off = view.data_ptr() - self.local.data_ptr()
        assert off >= 0 and off % view.element_size() == 0
        return off // view.element_size()


class _StoreComm:
    """CPU-side rendezvous of one process group over the c10d store (TCPStore): all-gather of small objects and a
    barrier.  Symmetric-memory set-up uses ONLY this — no NCCL kernel runs while buffers are being created and
    mapped (round 1 issued ~140 NCCL collectives there, next to cudaMalloc / IPC opens)."""

    _SEQ = {}

    def __init__(self, pg):
        import torch.distributed.distributed_c10d as c10d

        self.store = c10d._get_default_store()
        ranks = tuple(dist.get_process_group_ranks(pg if pg is not None else dist.group.WORLD))
        self.rank = dist.get_rank(pg)
        self.world = len(ranks)
        n = _StoreComm._SEQ.get(ranks, 0)          # construction is collective: same order on every member
        _StoreComm._SEQ[ranks] = n + 1
        self.prefix = "dtg/symm/" + "-".join(map(str, ranks)) + f"/{n}"
        self.seq = 0

    def all_gather(self, obj):
        import pickle

        k = f"{self.prefix}/ag{self.seq}"
        self.seq += 1
        self.store.set(f"{k}/{self.rank}", pickle.dumps(obj))
        return [pickle.loads(self.store.get(f"{k}/{r}")) for r in range(self.world)]

    def barrier(self):
        self.all_gather(None)


def _round_up(x, m):
    return (x + m - 1) // m * m


class _IpcChunk:
    """One cudaMalloc + (several ranks) one CUDA-IPC handle exchange: the single-rank case and the fallback when
    the system cannot export VMM allocations as file descriptors."""

    def __init__(self, group, nbytes):
        C = group.C
        self.raw, handle = C.symm_alloc(int(nbytes), group.device.index or 0)
        self.size = self.raw.numel()
        self.bases, self._opened = [], []
        handles = group.comm.all_gather(bytes(handle)) if group.world > 1 else [None]
        for r, h in enumerate(handles):
            if r == group.rank:
                self.bases.append(self.raw.data_ptr())
            else:
                p = C.symm_open(h, group.device.index or 0)
                self._opened.append(p)
                self.bases.append(p)
        self.mc_base = 0
        if group.world > 1:
            group.comm.barrier()
        self._C = C

    def local_view(self, off, n):
        return self._C.symm_alias(self.raw, int(off), int(n))   # NOT a slice: independent version counters

    def close(self):
        for p in self._opened:
            try:
                self._C.symm_close(p)
            except Exception:
                pass
        self._opened = []


class _VmmChunk:
    """(The reference never owns communication memory — NCCL registers whatever torch passes it, SURVEY.md §5.8.)
    One VMM chunk (``csrc/symm_vmm.cpp``): my physical allocation + every peer's, mapped side by side, and the
    NVLS multicast view.  File descriptors travel over an abstract Unix socket (SCM_RIGHTS); ordering over the store."""

    def __init__(self, group, nbytes):
        import socket
        import struct

        C, comm, world, rank = group.C, group.comm, group.world, group.rank
        self.chunk = C.VmmChunk(group.device.index or 0, int(nbytes), world, rank, group.multicast)
        self.size = int(self.chunk.size())
        my_fd = int(self.chunk.export_fd())
        mc_fd = int(self.chunk.mc_create_export()) if (group.multicast and rank == 0) else -1
        tag = f"{group.token}-{group._n_chunks}"
        addr = lambda r: f"\0dtg-symm-{tag}-{r}"  # noqa: E731  (abstract namespace: nothing to unlink)
        lst = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
        try:
            lst.bind(addr(rank))
            lst.listen(2 * world)
            comm.barrier()                                   # every listener exists
            for peer in range(world):
                if peer == rank:
                    continue
                with socket.socket(socket.AF_UNIX, socket.SOCK_STREAM) as c:
                    c.connect(addr(peer))
                    fds = [my_fd] + ([mc_fd] if mc_fd >= 0 else [])
                    socket.send_fds(c, [struct.pack("ii", rank, len(fds))], fds)
            for _ in range(world - 1):
                conn, _ = lst.accept()
                with conn:
                    msg, fds, _, _ = socket.recv_fds(conn, 8, 2)
                    peer, nfd = struct.unpack("ii", msg)
                    assert len(fds) == nfd, "file descriptors were lost in transit"
                    self.chunk.import_peer(peer, fds[0])
                    if nfd == 2:
                        self.chunk.mc_import(fds[1])
                    for fd in fds:
                        os.close(fd)
        finally:
            lst.close()
        os.close(my_fd)
        if mc_fd >= 0:
            os.close(mc_fd)
        self.chunk.map_all()
        self.mc_base = 0
        if group.multicast:
            self.chunk.mc_add_device()
            comm.barrier()                                   # every device joined the multicast team
            self.chunk.mc_bind_and_map()
            self.mc_base = int(self.chunk.mc_base())
        comm.barrier()                                       # every rank's memory is zeroed, mapped and bound
        base = int(self.chunk.base())
        self.bases = [base + r * self.size for r in range(world)]

    def local_view(self, off, n):
        return self.chunk.local_view(int(off), int(n))

    def close(self):
        self.chunk.release()


class SymmGroup:
    ALIGN = 4096                  # sub-allocation alignment inside a chunk (TMA / vector / shard alignment)
    FIRST_CHUNK = 64 << 20
    MAX_GROWTH = 4 << 30

    def __init__(self, device: torch.device, pg=None, ranks: Optional[List[int]] = None,
                 comm_blocks: Optional[int] = None):
        self.C = _ext.load(required=True)
        self.device = torch.device(device)
        self.pg = pg
        if dist.is_initialized() and (pg is not None or ranks is None):
            self.world = dist.get_world_size(pg)
            self.rank = dist.get_rank(pg)
        else:
            self.world, self.rank = 1, 0
        if self.world not in (1, 2, 4, 8):
            raise ValueError(f"symmetric collectives support 1/2/4/8 ranks, got {self.world}")
        if comm_blocks is None:
            # CTAs per collective kernel.  One rank: the fused kernel is a pure HBM-bound AdamW (14 B/element),
            # it needs the whole chip to reach memory bandwidth.  Several ranks: enough CTAs to keep
            # ~1 MB of 16-byte NVLink loads in flight (~2 us latency x ~800 GB/s) without starving the
            # tensor-core kernels it overlaps with.
            comm_blocks = int(os.environ.get("DTG_COMM_BLOCKS", 256 if self.world == 1 else 96))
        self.comm_blocks = min(comm_blocks, int(self.C.SYMM_MAX_CHANNELS))
        self.epoch = 0
        self._chunks, self._n_chunks, self._cur, self._used = [], 0, None, 0
        self.mode, self.multicast, self.comm, self.token = "local", False, None, ""
        if self.world > 1:
            # backend of the arena: VMM (fd export; + NVLS multicast when the fabric has it) or CUDA IPC
            self.comm = _StoreComm(pg)
            want = os.environ.get("DTG_SYMM", "vmm")
            fd_ok, mc_ok = self.C.vmm_support(self.device.index or 0)
            flags = self.comm.all_gather((bool(fd_ok) and want == "vmm", bool(mc_ok), os.getpid()))
            self.mode = "vmm" if all(f[0] for f in flags) else "ipc"
            self.multicast = (self.mode == "vmm" and all(f[1] for f in flags)
                              and os.environ.get("DTG_NVLS", "1") != "0")
            self.token = f"{flags[0][2]}-{self.comm.prefix.replace('/', '_')}"
        # multimem kernels (in-switch reduction) for the bucket collectives whenever the arena is multicast-bound
        self.nvls = self.multicast and os.environ.get("DTG_NVLS_KERNELS", "1") != "0"
        self.err = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.pads = self.alloc_bytes(int(self.C.SYMM_PAD_BYTES))
        self.pad_ptrs = self.pads.ptrs
        _LIVE_GROUPS.append(self)

    # -- allocation -----------------------------------------------------------------------------
    def _new_chunk(self, nbytes: int):
        if self.world == 1:
            ch = _IpcChunk(self, nbytes)
        else:
            ch = (_VmmChunk if self.mode == "vmm" else _IpcChunk)(self, nbytes)
        self._n_chunks += 1
        self._chunks.append(ch)
        self._cur, self._used = ch, 0
        return ch

    def reserve(self, nbytes: int):
        """Make room for ``nbytes`` of upcoming allocations in ONE chunk (one exchange) when the caller knows its
        total up front (the data-parallel engines do: parameters + gradients)."""
        if self.world > 1 and (self._cur is None or self._cur.size - self._used < nbytes):
            self._new_chunk(int(nbytes) + self.ALIGN)

    def alloc_bytes(self, nbytes: int) -> SymmBuffer:
        n = _round_up(max(int(nbytes), 1), self.ALIGN)
        if self.world == 1:
            ch = self._new_chunk(n)     # one rank: nothing to exchange, plain allocations
            off = 0
        else:
            if self._cur is None or self._cur.size - self._used < n:
                last = self._chunks[-1].size if self._chunks else 0
                self._new_chunk(max(n, min(max(self.FIRST_CHUNK, 2 * last), self.MAX_GROWTH)))
            ch, off = self._cur, self._used
            self._used += n
        raw = ch.local_view(off, n)
        ptrs = [b + off for b in ch.bases]
        return SymmBuffer(raw, ptrs, raw, mc_ptr=(ch.mc_base + off) if ch.mc_base else 0, handle=ch)

    def alloc(self, numel: int, dtype: torch.dtype) -> SymmBuffer:
        esize = torch.empty((), dtype=dtype).element_size()
        b = self.alloc_bytes(numel * esize)
        b.local = b._raw[: numel * esize].view(dtype)
        return b

    def allocator(self, registry: dict):
        """An ``alloc(n, dtype) -> tensor`` callable for ``flat.build_groups`` that records the
        SymmBuffer of each returned tensor in ``registry[data_ptr]``."""

        def alloc(n, dtype):
            b = self.alloc(n, dtype)
            registry[b.local.data_ptr()] = b
            return b.local

        return alloc

    def reserved_bytes(self) -> int:
        return sum(c.size for c in self._chunks)

    # -- collectives ------------------------------------------------------------------------------
    def _epochs(self, n: int = 2) -> int:
        e = self.epoch + 1
        self.epoch += n
        return e

    def allreduce_scale_(self, buf: SymmBuffer, elem_off: int, n: int, scale: float, blocks: Optional[int] = None):
        if self.nvls and buf.mc_ptr:
            self.C.comm_nvls_allreduce_scale(buf.mc_ptr, self.pad_ptrs, elem_off, n, scale, self.rank, self._epochs(2),
                                             self.err, blocks or self.comm_blocks)
            return
        self.C.comm_allreduce_scale(buf.ptrs, self.pad_ptrs, elem_off, n, scale, self.rank, self._epochs(2), self.err,
                                    blocks or self.comm_blocks)

    def rs_adamw_(self, grads: SymmBuffer, params: Optional[SymmBuffer], param_local, m, v, push_params: bool,
                  elem_off: int, n: int, hyper, step: int, grad_scale: float, blocks: Optional[int] = None):
        lr, b1, b2, eps, wd = hyper
        if self.nvls and grads.mc_ptr and (not push_params or (params is not None and params.mc_ptr)):
            # in-switch reduction of the gradient slice (+ multicast of the new parameters for ZeRO-1)
            self.C.comm_nvls_rs_adamw(grads.mc_ptr, params.mc_ptr if push_params else 0,
                                      params.ptrs[self.rank] if push_params else param_local.data_ptr(), m, v,
                                      push_params, self.pad_ptrs, elem_off, n, lr, b1, b2, eps, wd, step, grad_scale,
                                      self.rank, self._epochs(2), self.err, blocks or self.comm_blocks)
            return
        self.C.comm_rs_adamw(grads.ptrs, params.ptrs if params is not None else [], param_local, m, v, push_params,
                             self.pad_ptrs, elem_off, n, lr, b1, b2, eps, wd, step, grad_scale, self.rank,
                             self._epochs(2), self.err, blocks or self.comm_blocks)

    def allgather_(self, shards: SymmBuffer, full: torch.Tensor, shard_off: int, per: int, barrier: bool = True,
                   blocks: Optional[int] = None, copy_engine: bool = False):
        """``full[r*per:(r+1)*per] = shard of rank r``.  ``copy_engine=True``: a 1-warp barrier kernel + N async
        peer copies (zero SM time: the right choice for a prefetch that runs under GEMMs)."""
        self.C.comm_allgather(shards.ptrs, full, self.pad_ptrs, shard_off, per, self.rank, self._epochs(1), self.err,
                              barrier, 0 if copy_engine else (blocks or self.comm_blocks))

    def reduce_scatter_(self, grads: SymmBuffer, out: torch.Tensor, elem_off: int, n: int, scale: float,
                        blocks: Optional[int] = None):
        self.C.comm_reduce_scatter(grads.ptrs, out, self.pad_ptrs, elem_off, n, scale, self.rank, self._epochs(2),
                                   self.err, blocks or self.comm_blocks)

    # -- gradient clipping (csrc/grad_clip.cu) -------------------------------------------------------------------
    def reduce_sumsq_(self, buf: SymmBuffer, elem_off: int, n: int, scale: float, broadcast: bool,
                      ranges: torch.Tensor, partials: torch.Tensor, blocks: Optional[int] = None):
        """Reduce this rank's 1/N slice of ``buf`` (times ``scale``) and store it as bf16: into this rank's own buffer
        (``broadcast=False``, the reduce-scatter of ZeRO-1) or into every replica (``broadcast=True``, all-reduce).
        ``partials[b]`` = the sum of squares of the stored values CTA ``b`` wrote, over the element ``ranges``
        (int64 [R, 2] of [begin, end) relative to ``elem_off``) only."""
        blocks = blocks or self.comm_blocks
        if self.nvls and buf.mc_ptr:
            self.C.comm_nvls_reduce_sumsq(buf.mc_ptr, buf.ptrs[self.rank], self.pad_ptrs, elem_off, n, scale, broadcast,
                                          ranges, partials, self.rank, self._epochs(2), self.err, blocks)
            return
        self.C.comm_reduce_sumsq(buf.ptrs, self.pad_ptrs, elem_off, n, scale, broadcast, ranges, partials, self.rank,
                                 self._epochs(2), self.err, blocks)

    def clip_finalize_(self, partials: torch.Tensor, slots: SymmBuffer, parity: int, norm_scale: float,
                       max_norm: float, out: torch.Tensor):
        """``out[0]`` = sqrt(sum of every rank's ``partials``) * norm_scale, ``out[1]`` = the clip coefficient: the
        same bits on every rank (fixed-order fp64 sums, one device barrier)."""
        self.C.comm_clip_finalize(partials, slots.ptrs, self.pad_ptrs, parity, norm_scale, max_norm, out, self.rank,
                                  self._epochs(1), self.err)

    def barrier_(self):
        self.C.comm_barrier(self.pad_ptrs, self.rank, self._epochs(1), self.err)

    def check(self):
        """Raise if a device-side barrier timed out (a peer died or diverged)."""
        v = int(self.err.item())
        if v:
            raise RuntimeError(f"NVLink barrier timed out waiting for rank {v - 1} (group rank {self.rank}); "
                               + self.describe_pads())

    def describe_pads(self, timeout_s: float = 5.0) -> str:
        """Signal-pad state for a post-mortem: per peer, the range of epochs this rank has received over its
        channels, next to the epoch this rank's host has issued.  A peer stuck at a lower epoch never launched
        (or never finished) the matching collective.  The read runs on its own stream and gives up after
        ``timeout_s`` so it cannot itself hang behind a spinning kernel."""
        import time

        try:
            ch = int(self.C.SYMM_MAX_CHANNELS)
            mr = int(self.C.SYMM_PAD_BYTES) // 4 // ch           # uint32 [channels][max ranks]
            words = self.pads.local[: ch * mr * 4].view(torch.int32)
            host = torch.empty(ch * mr + 1, dtype=torch.int32, pin_memory=True)
            side = torch.cuda.Stream(device=self.device)
            done = torch.cuda.Event()
            with torch.cuda.stream(side):
                host[: ch * mr].copy_(words, non_blocking=True)
                host[ch * mr:].copy_(self.err, non_blocking=True)
                done.record(side)
            t0 = time.time()
            while not done.query():
                if time.time() - t0 > timeout_s:
                    return f"(pad read did not complete within {timeout_s:.0f} s; issued locally: {self.epoch})"
                time.sleep(0.01)
            tab = host[: ch * mr].view(ch, mr)[: self.comm_blocks, : self.world]
            seen = ", ".join(f"rank {p}: {int(tab[:, p].min())}..{int(tab[:, p].max())}" for p in range(self.world))
            return (f"epochs received per peer (min..max over {self.comm_blocks} channels): {seen}; "
                    f"issued locally: {self.epoch}; error flag: {int(host[ch * mr])}")
        except Exception as e:  # pragma: no cover - best effort diagnostics
            return f"(pad state unavailable: {e})"

    def close(self):
        for c in self._chunks:
            try:
                c.close()
            except Exception:
                pass
        self._chunks = []
        if self in _LIVE_GROUPS:
            _LIVE_GROUPS.remove(self)

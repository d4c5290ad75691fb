"""Federated communicator: one rank per GPU, clients round-robined over ranks, symmetric device arenas.

The reference has no communication layer at all ("network" = dict hand-off + ``torch.save``,
``experiment.py:189-203,233-241``). Here the exchange is the product:

* ``p2p``  (CUDA)  – every rank owns one symmetric arena that all peers map, and the collectives are the hand-written
  NVLink peer-memory kernels of ``csrc/fedcomm.cu``. The arena is built on the CUDA VMM API with an NVSwitch
  *multicast* view (``parallel/vmm.py``: ``multimem.ld_reduce`` / ``multimem.st`` = reduction / broadcast inside the
  switch, used by the FedAvg-style ``reduce_bcast``) when the box supports it, else ``cudaMalloc`` + CUDA IPC.
* ``nccl`` (CUDA)  – the *baseline harness*: the same API expressed with ``torch.distributed`` all-gathers plus local
  math. This is what the fused kernels are measured against; it is never used by the engine unless asked for.
* ``gloo`` (CPU)   – plumbing mode for world_size>1 without GPUs (tests, BASELINE config 1).
* ``local``        – world_size == 1 on CPU.

Buffers are *symmetric*: every rank performs the same sequence of allocations, so a buffer has the same offset in
every arena and a peer address is ``peer_base[rank] + offset``.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence

import torch
import torch.distributed as dist

from ..ops import native


@dataclass
class _Buf:
    name: str
    offset: int        # bytes from arena base
    n: int             # elements per slot
    slots: int         # slots per rank (clients per rank) or 1 for rank buffers
    dtype: torch.dtype
    per_client: bool


class _RawCuda:
    """Expose a raw device allocation to torch through ``__cuda_array_interface__``."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3,
                                         "strides": None}


def _dist_ready() -> bool:
    return dist.is_available() and dist.is_initialized()


def robust_aggregate(stack: torch.Tensor, rule: str, b: int = 0) -> torch.Tensor:
    """Coordinate-wise ``median`` / ``trimmed_mean`` of ``stack`` ``[K, n]`` (fp32) over its client dimension, with the
    ordering and arithmetic of ``fed_reduce_robust_kernel`` (see ``FedComm.reduce_robust``)."""
    K = stack.shape[0]
    s = torch.sort(stack, dim=0, stable=True).values
    if rule == "median":
        if K % 2:
            return s[(K - 1) // 2].clone()
        return s[K // 2 - 1] * 0.5 + s[K // 2] * 0.5
    acc = torch.full_like(s[0], -0.0)                 # (-0.0 is the exact identity of the addition)
    for t in range(b, K - b):
        acc = acc + s[t]
    return acc / torch.full_like(acc, float(K - 2 * b))  # (a true division, also on CUDA)


class FedComm:
    def __init__(self, device: torch.device | str, num_clients: int, arena_bytes: int = 1 << 30,
                 mode: Optional[str] = None, timeout_s: float = 30.0, comm_blocks: int = 0, group=None):
        self.device = torch.device(device)
        if self.device.type == "cuda" and self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.group = group
        self.rank = dist.get_rank(group) if _dist_ready() else 0
        self.world = dist.get_world_size(group) if _dist_ready() else 1
        self.K = int(num_clients)
        self.slots = (self.K + self.world - 1) // self.world
        if mode is None:
            mode = "p2p" if self.device.type == "cuda" else ("gloo" if self.world > 1 else "local")
        self.mode = mode
        self.timeout_s = float(timeout_s)
        self.arena_bytes = int(arena_bytes)
        self.bufs: Dict[str, _Buf] = {}
        self._cursor = 0
        self._peer_base: List[int] = []
        self._keep = []
        self.bytes_moved = 0          # algorithmic NVLink/peer bytes pulled+pushed by this rank
        self.nvls = True              # use the multicast (in-switch) reduce when the arena has a multicast view
        self.nvls_min_bytes = 1 << 20
        self.nvls_launches = 0
        self.block_cap = 0            # > 0: upper bound on the grid of the collectives launched while it is set
        self._mc_base = 0
        self._vmm = None
        self.backend = mode
        if self.mode == "p2p":
            self._init_p2p()
            self.comm_blocks = comm_blocks or 132 * 2
        else:
            self._arena = torch.zeros(self.arena_bytes, dtype=torch.uint8, device=self.device)
            self.comm_blocks = 0

    # ------------------------------------------------------------------ placement
    def owner(self, client: int) -> int:
        return client % self.world

    def slot(self, client: int) -> int:
        return client // self.world

    def local_clients(self) -> List[int]:
        return [c for c in range(self.K) if self.owner(c) == self.rank]

    # ------------------------------------------------------------------ arena
    def _init_p2p(self) -> None:
        import os
        lib = native.load()
        self._lib = lib
        if lib.flpr_comm_max_ranks() < self.world:
            raise native.NativeError(f"world size {self.world} exceeds MAX_RANKS")
        if lib.flpr_comm_max_clients() < self.K:
            raise native.NativeError(f"{self.K} clients exceed MAX_CLIENTS")
        torch.cuda.set_device(self.device)
        self._flag_bytes = ((lib.flpr_comm_flag_page_bytes() + 4095) // 4096) * 4096
        self._cursor = self._flag_bytes
        self._vmm = None
        self._mc_base = 0
        self.backend = "ipc"
        self.backend_note = ""
        if self.world > 1 and os.environ.get("FLPR_COMM_VMM", "1") != "0":
            # VMM arena + NVSwitch multicast view; any failure (every rank takes the same branch: the decision is
            # all-reduced) leaves the cudaMalloc + IPC arena below
            from .vmm import SymmetricVmm
            err = None
            try:
                vmm = SymmetricVmm(self.device, self.arena_bytes, self.rank, self.world, self.group,
                                   multicast=os.environ.get("FLPR_COMM_NVLS", "1") != "0")
            except Exception as ex:  # noqa: BLE001  (driver / cuda-python / fabric problems of any kind)
                vmm, err = None, f"{type(ex).__name__}: {ex}"
            ok = torch.tensor([0 if vmm is None else 1], device=self.device)
            dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=self.group)
            if ok.item():
                self._vmm = vmm
                self.arena_bytes = vmm.size
                self._base = vmm.base
                self._peer_base = list(vmm.peer_base)
                self._mc_base = vmm.mc_base
                self.backend = "vmm+nvls" if vmm.mc_base else "vmm"
                self.backend_note = getattr(vmm, "mc_error", "")
            else:
                if vmm is not None:
                    vmm.close()
                self.backend_note = err or "a peer rank could not build the VMM arena"
        if self._vmm is None:
            base = C.c_void_p()
            native.check(lib.flpr_symm_alloc(C.byref(base), self.arena_bytes), "flpr_symm_alloc")
            self._base = base.value
        self._arena = torch.as_tensor(_RawCuda(self._base, self.arena_bytes), device=self.device)
        if self._vmm is not None:
            self._arena.zero_()
            torch.cuda.synchronize(self.device)
            dist.barrier(group=self.group)
        elif self.world > 1:
            handle = (C.c_ubyte * 64)()
            native.check(lib.flpr_ipc_get_handle(C.c_void_p(self._base), handle), "flpr_ipc_get_handle")
            handles: List[Optional[bytes]] = [None] * self.world
            dist.all_gather_object(handles, bytes(handle), group=self.group)
            for r in range(self.world):
                if r == self.rank:
                    self._peer_base.append(self._base)
                else:
                    p = C.c_void_p()
                    buf = (C.c_ubyte * 64).from_buffer_copy(handles[r])
                    native.check(lib.flpr_ipc_open_handle(buf, C.byref(p)), f"flpr_ipc_open_handle(rank {r})")
                    self._peer_base.append(p.value)
            dist.barrier(group=self.group)
        else:
            self._peer_base = [self._base]
        self._flag_pages = (C.c_void_p * self.world)(*[C.c_void_p(b) for b in self._peer_base])
        # host-mapped mailbox mirroring the watchdog's error word: polled after every collective without a CUDA call
        self._mailbox = torch.zeros(4, dtype=torch.int32).pin_memory()
        native.check(lib.flpr_comm_set_mailbox(C.c_void_p(self._base), C.c_void_p(self._mailbox.data_ptr())),
                     "flpr_comm_set_mailbox")

    def _stream(self):
        """Stream handle the collectives are launched on (the calling thread's current CUDA stream)."""
        return native.stream(self.device)

    def set_channel(self, channel: int) -> None:
        """Flag channel of the collectives launched by the calling thread from now on (concurrent collectives - one
        on a communication stream, one on the compute stream - must use different channels; same choice on every
        rank)."""
        if self.mode == "p2p":
            native.check(self._lib.flpr_comm_set_channel(int(channel)), "flpr_comm_set_channel")

    def close(self) -> None:
        if self.mode == "p2p" and getattr(self, "_base", None):
            torch.cuda.synchronize(self.device)
            if self.world > 1:
                dist.barrier(group=self.group)
            self._arena = None
            if self._vmm is not None:
                self._vmm.close()
                self._vmm = None
            else:
                for r, p in enumerate(self._peer_base):
                    if r != self.rank:
                        self._lib.flpr_ipc_close(C.c_void_p(p))
                self._lib.flpr_symm_free(C.c_void_p(self._base))
            self._base = None

    def _alloc(self, name: str, n: int, slots: int, dtype: torch.dtype, per_client: bool) -> _Buf:
        if name in self.bufs:
            b = self.bufs[name]
            assert (b.n, b.slots, b.dtype) == (n, slots, dtype), f"buffer {name} re-declared with a different shape"
            return b
        item = torch.empty((), dtype=dtype).element_size()
        assert (n * item) % 16 == 0, "symmetric buffers must be multiples of 16 bytes per slot"
        nbytes = n * item * slots
        off = (self._cursor + 255) // 256 * 256
        if off + nbytes > self.arena_bytes:
            raise MemoryError(f"symmetric arena exhausted allocating {name}: need {off + nbytes} of {self.arena_bytes}")
        self._cursor = off + nbytes
        b = _Buf(name, off, n, slots, dtype, per_client)
        self.bufs[name] = b
        return b

    def alloc_client_buffer(self, name: str, n: int, dtype: torch.dtype = torch.float32) -> None:
        """One slot of ``n`` elements for every client (``ceil(K/world)`` slots per rank)."""
        self._alloc(name, n, self.slots, dtype, True)

    def alloc_rank_buffer(self, name: str, n: int, dtype: torch.dtype = torch.float32) -> None:
        self._alloc(name, n, 1, dtype, False)

    def _view(self, b: _Buf, slot: int) -> torch.Tensor:
        item = torch.empty((), dtype=b.dtype).element_size()
        start = b.offset + slot * b.n * item
        return self._arena[start:start + b.n * item].view(b.dtype)

    def client_view(self, name: str, client: int) -> torch.Tensor:
        assert self.owner(client) == self.rank, f"client {client} is not hosted on rank {self.rank}"
        return self._view(self.bufs[name], self.slot(client))

    def rank_view(self, name: str) -> torch.Tensor:
        return self._view(self.bufs[name], 0)

    def _addr(self, b: _Buf, rank: int, slot: int) -> int:
        item = torch.empty((), dtype=b.dtype).element_size()
        return self._peer_base[rank] + b.offset + slot * b.n * item

    def _client_ptrs(self, name: str, clients: Sequence[int]):
        b = self.bufs[name]
        arr = (C.c_void_p * len(clients))(*[C.c_void_p(self._addr(b, self.owner(c), self.slot(c))) for c in clients])
        return arr

    def _rank_ptrs(self, name: str):
        b = self.bufs[name]
        return (C.c_void_p * self.world)(*[C.c_void_p(self._addr(b, r, 0)) for r in range(self.world)])

    def _grid_for(self, nbytes: int) -> int:
        """Grid size of a collective moving ``nbytes`` per rank. Every block takes part in the cross-rank barriers (and
        spins while a peer is late), so small buffers use few blocks; ``self.block_cap`` (set around a collective that
        runs next to compute kernels) bounds the SM footprint of the spinning. Block b of one rank pairs with block b
        of every peer, so ``nbytes`` (and ``block_cap``) MUST be computed from rank-invariant quantities only - never
        from how many clients this rank happens to host."""
        want = max(4, (int(nbytes) + (256 << 10) - 1) // (256 << 10))
        cap = self.block_cap or self.comm_blocks
        return int(min(want, cap, self.comm_blocks))

    def _remote(self, clients: Sequence[int]) -> int:
        return sum(1 for c in clients if self.owner(c) != self.rank)

    # ------------------------------------------------------------------ gather helper for non-p2p modes
    def _gather_clients(self, name: str, clients: Sequence[int]) -> torch.Tensor:
        """[len(clients), n] on every rank via a library all-gather (baseline / CPU modes)."""
        b = self.bufs[name]
        local = torch.stack([self._view(b, s) for s in range(b.slots)]).contiguous()      # [slots, n]
        if self.world == 1:
            allb = local
        else:
            allb = torch.empty((self.world * b.slots, b.n), dtype=local.dtype, device=local.device)
            dist.all_gather_into_tensor(allb, local, group=self.group)
        return torch.stack([allb[self.owner(c) * b.slots + self.slot(c)] for c in clients])

    _TIMEOUT_MSG = ("a flpr collective timed out waiting for a peer rank (flag watchdog fired); the kernels skipped "
                    "their store phase, no partial aggregate was published")

    def poll_errors(self) -> None:
        """Non-blocking: raise as soon as a *completed* collective has reported a missed barrier (host-mapped mailbox,
        no CUDA call, no device sync). Called after every collective launch and at the round boundaries."""
        if self.mode == "p2p" and int(self._mailbox[0]) != 0:
            raise native.NativeError(self._TIMEOUT_MSG)

    def check_errors(self) -> None:
        """Blocking: reads the device-side error word (synchronises the device)."""
        if self.mode != "p2p":
            return
        err = C.c_int(0)
        self._lib.flpr_comm_read_error(C.c_void_p(self._base), C.byref(err))
        if err.value or int(self._mailbox[0]) != 0:
            raise native.NativeError(self._TIMEOUT_MSG)

    # ------------------------------------------------------------------ collectives
    def barrier(self) -> None:
        if self.mode == "p2p":
            rc = self._lib.flpr_comm_barrier(self.rank, self.world, self._flag_pages, self.timeout_s,
                                             self._stream())
            native.check(rc, "flpr_comm_barrier")
            native.count_launch()
        elif self.world > 1:
            dist.barrier(group=self.group)

    def reduce_bcast(self, src: str, dst: str, clients: Sequence[int], cnt: Optional[str] = None,
                     weights: Optional[Sequence[float]] = None) -> None:
        """C1+C2: ``dst = sum_c w_c * src_c`` on every rank; ``w_c = cnt_c / sum(cnt)`` when ``cnt`` names a
        per-client scalar buffer (FedAvg ``train_cnt`` weighting, ``methods/fedavg.py:386-397``)."""
        bs, bd = self.bufs[src], self.bufs[dst]
        assert bs.n == bd.n and bs.dtype == torch.float32 and bd.dtype == torch.float32
        if self.mode == "p2p" and self._mc_base and self.nvls and bs.n * 4 > self.nvls_min_bytes:
            # the kernel choice must be the same on every rank: decide on the largest number of participants hosted
            # by ANY rank, not on how many this rank hosts
            per_rank = [0] * self.world
            for c in clients:
                per_rank[self.owner(c)] += 1
            if max(per_rank) <= self._lib.flpr_comm_max_local():
                mine = [c for c in clients if self.owner(c) == self.rank]
                return self._reduce_bcast_nvls(src, dst, clients, mine, cnt, weights)
        if self.mode == "p2p":
            srcp = self._client_ptrs(src, clients)
            cntp = self._client_ptrs(cnt, clients) if cnt is not None else None
            wv = (C.c_float * len(clients))(*[float(x) for x in weights]) if weights is not None else None
            rc = self._lib.flpr_comm_reduce_bcast(self.rank, self.world, self._flag_pages, self.timeout_s, len(clients),
                                                  srcp, cntp, wv, self._rank_ptrs(dst), bs.n,
                                                  self._grid_for(bs.n * 4 * max(len(clients), 1) // max(self.world, 1)),
                                                  self._stream())
            native.check(rc, "flpr_comm_reduce_bcast")
            native.count_launch()
            self.poll_errors()
            share = bs.n * 4 / self.world
            self.bytes_moved += int(share * self._remote(clients) + share * (self.world - 1))
            return
        stack = self._gather_clients(src, clients).float()
        if cnt is not None:
            w = self._gather_clients(cnt, clients)[:, 0].float()
            w = w / w.sum()
        else:
            w = torch.tensor(list(weights), dtype=torch.float32, device=stack.device)
        self.rank_view(dst).copy_((w[:, None] * stack).sum(0))

    ROBUST_RULES = ("median", "trimmed_mean")       # index = the ``rule`` code of ``flpr_comm_reduce_robust``

    def reduce_robust(self, src: str, dst: str, clients: Sequence[int], rule: str, b: int = 0) -> None:
        """C1+C2, Byzantine-robust: ``dst`` = coordinate-wise ``median`` or ``trimmed_mean`` of the uploads of ``clients``
        on every rank, unweighted. Per coordinate the K values are ordered by ``(value, position in clients)`` (NaN
        above +inf, -0.0 == +0.0), i.e. a stable sort. ``median``: the middle value, or ``0.5 * lo + 0.5 * hi`` of the
        two middle values for even K. ``trimmed_mean``: the mean of sorted positions ``[b, K - b)``, summed in fp32 in
        ascending order. ``p2p`` runs ``fed_reduce_robust_kernel`` (two-shot; never the NVLS path, whose in-switch sums
        cannot form order statistics); the other modes all-gather and sort."""
        bs, bd = self.bufs[src], self.bufs[dst]
        assert bs.n == bd.n and bs.dtype == torch.float32 and bd.dtype == torch.float32
        if rule not in self.ROBUST_RULES:
            raise ValueError(f"reduce_robust: unknown rule {rule!r} (one of {self.ROBUST_RULES})")
        K, b = len(clients), int(b)
        if not (b == 0 if rule == "median" else 0 <= 2 * b < K):
            raise ValueError(f"reduce_robust: b = {b} out of range for {rule!r} with {K} clients")
        if self.mode == "p2p":
            rc = self._lib.flpr_comm_reduce_robust(self.rank, self.world, self._flag_pages, self.timeout_s, K,
                                                   self._client_ptrs(src, clients), self._rank_ptrs(dst),
                                                   self.ROBUST_RULES.index(rule), b, bs.n,
                                                   self._grid_for(bs.n * 4 * max(K, 1) // max(self.world, 1)),
                                                   self._stream())
            native.check(rc, "flpr_comm_reduce_robust")
            native.count_launch()
            self.poll_errors()
            share = bs.n * 4 / self.world
            self.bytes_moved += int(share * self._remote(clients) + share * (self.world - 1))
            return
        self.rank_view(dst).copy_(robust_aggregate(self._gather_clients(src, clients).float(), rule, b))

    def _reduce_bcast_nvls(self, src, dst, clients, mine, cnt, weights) -> None:
        """C1+C2 through the switch: local fold of this rank's clients -> ``multimem.ld_reduce`` of the partials for
        this rank's slice -> scale -> ``multimem.st`` into every rank's destination (``fed_reduce_bcast_nvls``)."""
        bs, bd = self.bufs[src], self.bufs[dst]
        pname = f"_nvls_partial_{bs.n}"
        if pname not in self.bufs:
            self.alloc_rank_buffer(pname, bs.n)              # symmetric: every rank reaches this line in the same call
        bp = self.bufs[pname]
        srcp = self._client_ptrs(src, mine) if mine else None
        cntp = self._client_ptrs(cnt, mine) if (cnt is not None and mine) else None
        cnt_all = self._client_ptrs(cnt, clients) if cnt is not None else None
        wv, w_total = None, 0.0
        if cnt is None:
            wmap = {c: float(w) for c, w in zip(clients, weights)}
            w_total = 1.0                                    # explicit weights are used as given (not re-normalised)
            wv = (C.c_float * max(len(mine), 1))(*[wmap[c] for c in mine]) if mine else None
        rc = self._lib.flpr_comm_reduce_bcast_nvls(
            self.rank, self.world, self._flag_pages, self.timeout_s, len(mine), srcp, cntp, wv, len(clients), cnt_all,
            w_total, C.c_void_p(self._addr(bp, self.rank, 0)), C.c_void_p(self._mc_base + bp.offset),
            C.c_void_p(self._mc_base + bd.offset), bs.n, self._grid_for(bs.n * 4 * len(clients) // self.world),
            self._stream())
        native.check(rc, "flpr_comm_reduce_bcast_nvls")
        native.count_launch()
        self.poll_errors()
        self.nvls_launches += 1
        share = bs.n * 4 / self.world
        self.bytes_moved += int(share * (self.world - 1) * 2)     # pulled through the switch + multicast out

    def mix(self, src: str, clients: Sequence[int], rows: torch.Tensor, local_clients: Sequence[int],
            dst_g: Optional[Sequence[torch.Tensor]] = None, dst_theta: Optional[Sequence[torch.Tensor]] = None,
            dst_bf16: Optional[Sequence[torch.Tensor]] = None) -> None:
        """C4: for every local client ``i``: ``out_i = sum_j rows[i, j] * src_j`` written to ``dst_g[i]``,
        ``dst_theta[i]`` (fp32) and ``dst_bf16[i]`` in one pass. ``rows``: ``[len(local_clients), len(clients)]``."""
        bs = self.bufs[src]
        L = len(local_clients)
        if L == 0 and self.mode != "p2p":
            if self.world > 1:
                self._gather_clients(src, clients)  # keep the collective sequence aligned
            return
        if self.mode == "p2p":
            rows_dev = rows.detach().float().contiguous() if rows.is_cuda else None
            rows_h = None if rows_dev is not None else rows.detach().float().cpu().contiguous()
            max_l = self._lib.flpr_comm_max_local()
            srcp = self._client_ptrs(src, clients)
            # every rank issues the same number of launches (the kernels barrier across ranks)
            n_launch = (self.slots + max_l - 1) // max_l
            for it in range(n_launch):
                idx = list(range(it * max_l, min((it + 1) * max_l, L)))
                wv, wd = None, None
                if idx and rows_dev is not None:
                    wd = rows_dev[idx[0]:idx[-1] + 1]
                    self._keep = [wd]
                elif idx:
                    wv = (C.c_float * (len(idx) * len(clients)))(*rows_h[idx].reshape(-1).tolist())

                def arr(lst):
                    if lst is None or not idx:
                        return None
                    return (C.c_void_p * len(idx))(*[C.c_void_p(lst[i].data_ptr()) for i in idx])

                rc = self._lib.flpr_comm_mix(self.rank, self.world, self._flag_pages, self.timeout_s, len(clients),
                                             len(idx), srcp, wv, native.ptr(wd), arr(dst_g), arr(dst_theta),
                                             arr(dst_bf16), bs.n,
                                             self._grid_for(bs.n * 4 * len(clients)), self._stream())
                native.check(rc, "flpr_comm_mix")
                native.count_launch()
                self.poll_errors()
                if idx:
                    self.bytes_moved += int(bs.n * 4 * self._remote(clients))
            return
        stack = self._gather_clients(src, clients).float()
        out = rows.detach().float().to(stack.device) @ stack
        for i in range(L):
            if dst_g is not None:
                dst_g[i].view(-1).copy_(out[i])
            if dst_theta is not None:
                dst_theta[i].view(-1).copy_(out[i])
            if dst_bf16 is not None:
                dst_bf16[i].view(-1).copy_(out[i])

    def curv_moments(self, fisher: str, param: str, clients: Sequence[int], dst_f: str, dst_fp: str, dst_fpp: str
                     ) -> None:
        """C3: ``sum_j F_j``, ``sum_j F_j p_j``, ``sum_j F_j p_j^2`` into three rank buffers on every rank."""
        bf = self.bufs[fisher]
        if self.mode == "p2p":
            rc = self._lib.flpr_comm_curv_moments(self.rank, self.world, self._flag_pages, self.timeout_s, len(clients),
                                                  self._client_ptrs(fisher, clients), self._client_ptrs(param, clients),
                                                  self._rank_ptrs(dst_f), self._rank_ptrs(dst_fp),
                                                  self._rank_ptrs(dst_fpp), bf.n,
                                                  self._grid_for(2 * bf.n * 4 * max(len(clients), 1) // max(self.world, 1)),
                                                  self._stream())
            native.check(rc, "flpr_comm_curv_moments")
            native.count_launch()
            self.poll_errors()
            share = bf.n * 4 / self.world
            self.bytes_moved += int(2 * share * self._remote(clients) + 3 * share * (self.world - 1))
            return
        Fs = self._gather_clients(fisher, clients).float()
        Ps = self._gather_clients(param, clients).float()
        self.rank_view(dst_f).copy_(Fs.sum(0))
        self.rank_view(dst_fp).copy_((Fs * Ps).sum(0))
        self.rank_view(dst_fpp).copy_((Fs * Ps * Ps).sum(0))

    def gather_strided(self, src: str, clients: Sequence[int], out: torch.Tensor) -> None:
        """C5/C6: ``out[e, j] = src_{clients[j]}[e]`` (trailing client dim), ``out`` local ``[n, len(clients)]``."""
        bs = self.bufs[src]
        assert out.is_contiguous() and out.numel() == bs.n * len(clients)
        if self.mode == "p2p":
            rc = self._lib.flpr_comm_gather_strided(self.rank, self.world, self._flag_pages, self.timeout_s,
                                                    len(clients), self._client_ptrs(src, clients), native.ptr(out),
                                                    bs.n, self._grid_for(bs.n * 4 * len(clients)),
                                                    self._stream())
            native.check(rc, "flpr_comm_gather_strided")
            native.count_launch()
            self.poll_errors()
            self.bytes_moved += int(bs.n * 4 * self._remote(clients))
            return
        stack = self._gather_clients(src, clients).float()
        out.view(bs.n, len(clients)).copy_(stack.t())

    def pull(self, src: str, client: int, dst: Optional[torch.Tensor] = None,
             dst_bf16: Optional[torch.Tensor] = None) -> None:
        """C2: copy client ``client``'s slot of ``src`` (wherever it lives) into local tensors (fp32 and/or bf16)."""
        bs = self.bufs[src]
        if self.mode == "p2p":
            addr = self._addr(bs, self.owner(client), self.slot(client))
            rc = self._lib.flpr_comm_pull_copy(self.rank, self.world, self._flag_pages, self.timeout_s,
                                               C.c_void_p(addr), native.ptr(dst), native.ptr(dst_bf16), bs.n,
                                               self._grid_for(bs.n * 4), self._stream())
            native.check(rc, "flpr_comm_pull_copy")
            native.count_launch()
            self.poll_errors()
            if self.owner(client) != self.rank:
                self.bytes_moved += bs.n * 4
            return
        row = self._gather_clients(src, [client])[0]
        if dst is not None:
            dst.view(-1).copy_(row)
        if dst_bf16 is not None:
            dst_bf16.view(-1).copy_(row)

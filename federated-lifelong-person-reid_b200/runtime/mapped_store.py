"""Checkpoint files as persistent, CUDA-registered file mappings: a snapshot is a set of DMAs straight into the file.

The asynchronous :class:`~.checkpoint.CheckpointStore` moves a snapshot device -> pinned arena -> writer process ->
``torch.save`` -> fresh RAM-disk pages. The federated round produces several GB of reference-layout files, and at
8 GPUs the *host* side of that pipeline (page allocation + one CPU copy per byte) can bound the round. Here the host
CPU does not touch the payload at all:

* The byte layout of a checkpoint file is a pure function of the state's *structure* (keys, shapes, dtypes): the
  legacy ``torch.save`` container is ``[pickles: magic, protocol, sys-info, object graph, storage keys]`` followed by
  ``[int64 numel][raw bytes]`` per storage; all tensors of one dtype are laid out as views of ONE storage, so the data
  region is contiguous per dtype. :func:`legacy_layout` emits those pickles itself (tensors reduce to
  ``_rebuild_tensor_v2`` over persistent storage ids, exactly what ``torch.load`` expects) and pads the storage-key
  pickle with an ignored junk string so that the data region starts at a fixed offset even when scalars in the object
  graph (``train_cnt``) change their encoded width from round to round.
* The file is created once, ``mmap``-ed ``MAP_SHARED`` and page-locked with ``cudaHostRegister``. Saving = (a) the
  tensors are gathered into a *device-resident image* of the file's data region by one multi-tensor copy on the
  producing stream - the snapshot is taken at that instant, the sources may be overwritten right away, no fence on the
  compute stream ever waits for PCIe - and (b) ONE ``cudaMemcpyAsync`` of the image into the mapping on a copy stream.
  The pickle prefix is re-emitted only when a scalar in the object graph changed. No byte of payload is pickled,
  staged in host memory or copied by a CPU.
* Files whose name is unique per round (``{round}-{src}-{dst}.ckpt``) recycle the mappings of rounds that have left
  the retention window (``engine_opts.payload_ring``; 0 = keep every round like the reference, allocating fresh
  mappings): the old file is renamed to the new name and overwritten in place.
* FedSTIL's exemplar file keeps the reference schema ``{np.int64 pid: [(ndarray, class_id), ...]}``
  (``methods/fedstil.py:841,846``): its pickle is laid out once per exemplar-set structure and the fp32 prototypes are
  DMA-ed to the recorded array offsets.

Only page-cache-less file systems qualify (tmpfs / ramfs: device DMA does not mark pages dirty, a disk-backed file
would never be written back); anything else falls back to the staged pipeline of the parent class. On the CPU the
same layout code runs with plain ``memcpy`` - that is what the CPU test-suite exercises.
"""
from __future__ import annotations

import collections
import ctypes as C
import io
import mmap
import os
import pickle
import re
import threading
from typing import Any, Dict, List, Optional, Tuple

import torch

from .checkpoint import CheckpointStore, _dedicated_stream

_PAYLOAD_NAME = re.compile(r"^\d+-")          # '{round}-{src}-{dst}': unique per round
_SLACK = 512                                  # bytes of padding available for growing scalars


# ===================================================================================================== layout
class _StorageRef:
    __slots__ = ("key", "dtype", "numel")

    def __init__(self, key: str, dtype: torch.dtype, numel: int):
        self.key, self.dtype, self.numel = key, dtype, numel


def _storage_type(dtype: torch.dtype):
    """The legacy typed-storage class ``torch.load`` expects in a persistent id (``torch.FloatStorage`` ...)."""
    return getattr(torch, torch.storage._dtype_to_storage_type_map()[dtype])


class _Segment:
    __slots__ = ("tensor", "offset", "nbytes")

    def __init__(self, tensor: torch.Tensor, offset: int, nbytes: int):
        self.tensor, self.offset, self.nbytes = tensor, offset, nbytes


class Layout:
    """Byte layout of one checkpoint file: ``prefix`` (pickles, padded to ``data_start``) + storages."""

    def __init__(self, signature, data_start: int, segments: List[_Segment], total: int, headers: List[Tuple[int, int]]):
        self.signature = signature
        self.data_start = data_start
        self.segments = segments
        self.total = total
        self.headers = headers              # (offset, numel) of the 8-byte storage headers


def _signature(obj: Any):
    """Structure of a state: everything that determines the byte layout except scalar values."""
    if isinstance(obj, torch.Tensor):
        return ("T", tuple(obj.shape), str(obj.dtype))
    if isinstance(obj, dict):
        return ("D", type(obj).__name__, tuple((repr(k), _signature(v)) for k, v in obj.items()))
    if isinstance(obj, (list, tuple)):
        return ("L", type(obj).__name__, tuple(_signature(v) for v in obj))
    if isinstance(obj, (bool, int, float, type(None))):
        return ("S", type(obj).__name__)
    if isinstance(obj, str):
        return ("s", len(obj.encode()))
    return ("O", type(obj).__name__, len(pickle.dumps(obj, protocol=2)))


def _has_foreign(obj: Any) -> bool:
    """True when the state holds bulk data that is not a tensor (numpy arrays: iCaRL's exemplar images in the
    reference schema). Such states keep the staged pipeline - their payload lives inside the pickle itself."""
    stack = [obj]
    while stack:
        o = stack.pop()
        if isinstance(o, (torch.Tensor, bool, int, float, str, type(None))):
            continue
        if isinstance(o, dict):
            stack.extend(o.keys())
            stack.extend(o.values())
        elif isinstance(o, (list, tuple)):
            stack.extend(o)
        else:
            nbytes = getattr(o, "nbytes", None)
            if nbytes is None or nbytes > 64:
                return True
    return False


def _scalars(obj: Any):
    """The non-tensor leaves of a state (what the pickle prefix depends on besides the structure)."""
    if isinstance(obj, torch.Tensor):
        return None
    if isinstance(obj, dict):
        return tuple(_scalars(v) for v in obj.values())
    if isinstance(obj, (list, tuple)):
        return tuple(_scalars(v) for v in obj)
    if isinstance(obj, (bool, int, float, str, type(None))):
        return obj
    return pickle.dumps(obj, protocol=2)


def _tensors_in_order(obj: Any, out: List[torch.Tensor], seen: Dict[int, bool]) -> None:
    """Tensors in the order the pickler meets them (dict insertion order, depth first), shared objects once."""
    if isinstance(obj, torch.Tensor):
        if id(obj) not in seen:
            seen[id(obj)] = True
            out.append(obj)
    elif isinstance(obj, dict):
        for v in obj.values():
            _tensors_in_order(v, out, seen)
    elif isinstance(obj, (list, tuple)):
        for v in obj:
            _tensors_in_order(v, out, seen)


def _rebind(layout: "Layout", state: Any) -> "Layout":
    """The same byte layout pointing at the tensors of a new state of identical structure."""
    ts: List[torch.Tensor] = []
    _tensors_in_order(state, ts, {})
    if len(ts) != len(layout.segments):
        raise ValueError("state does not match the cached layout")
    by_dtype: Dict[torch.dtype, List[torch.Tensor]] = {}
    for t in ts:                                            # file order: dtypes by first appearance, tensors in order
        by_dtype.setdefault(t.dtype, []).append(t)
    ts = [t for group in by_dtype.values() for t in group]
    if any(t.numel() * t.element_size() != seg.nbytes for t, seg in zip(ts, layout.segments)):
        raise ValueError("state does not match the cached layout")
    segs = [_Segment(t, seg.offset, seg.nbytes) for t, seg in zip(ts, layout.segments)]
    return Layout(layout.signature, layout.data_start, segs, layout.total, layout.headers)


def _main_pickle(state: Any) -> Tuple[bytes, List[Tuple[_StorageRef, List[Tuple[torch.Tensor, int]]]]]:
    """The object-graph pickle of the legacy container. All tensors of one dtype are views of ONE storage (a tensor is
    ``_rebuild_tensor_v2(storage, element offset, size, contiguous strides)``): the file then holds a single
    ``[numel][data]`` record per dtype, i.e. the data region is contiguous - one DMA per dtype, no record headers in
    between. Returns the bytes and ``[(storage, [(tensor, element offset), ...]), ...]`` in file order."""
    def run(numels: Optional[Dict[torch.dtype, int]]):
        groups: Dict[torch.dtype, Tuple[_StorageRef, List[Tuple[torch.Tensor, int]]]] = {}
        by_id: Dict[int, Tuple[_StorageRef, int]] = {}
        buf = io.BytesIO()

        class P(pickle.Pickler):
            def persistent_id(self, obj):                                   # noqa: D401
                if isinstance(obj, _StorageRef):
                    return ("storage", _storage_type(obj.dtype), obj.key, "cpu", obj.numel, None)
                return None

            def reducer_override(self, obj):
                if isinstance(obj, torch.Tensor):
                    hit = by_id.get(id(obj))
                    if hit is None:
                        g = groups.get(obj.dtype)
                        if g is None:
                            ref = _StorageRef(str(len(groups)), obj.dtype, numels[obj.dtype] if numels else 0)
                            g = groups[obj.dtype] = (ref, [])
                        off = sum(t.numel() for t, _ in g[1][-1:]) + (g[1][-1][1] if g[1] else 0)
                        g[1].append((obj, off))
                        hit = by_id[id(obj)] = (g[0], off)
                    stride, acc = [], 1
                    for d in reversed(obj.shape):
                        stride.append(acc)
                        acc *= max(int(d), 1)
                    return (torch._utils._rebuild_tensor_v2,
                            (hit[0], hit[1], tuple(obj.shape), tuple(reversed(stride)), False, collections.OrderedDict()))
                return NotImplemented

        P(buf, protocol=2).dump(state)
        return buf.getvalue(), list(groups.values())

    _, groups = run(None)                                   # pass 1: which tensors, how many elements per dtype
    numels = {ref.dtype: (members[-1][1] + members[-1][0].numel() if members else 0) for ref, members in groups}
    return run(numels)                                      # pass 2: the real pickle (storage sizes are part of it)


_HEAD: Optional[bytes] = None


def _head_pickles() -> bytes:
    """magic number, protocol version, sys-info: the three leading pickles of the legacy container."""
    global _HEAD
    if _HEAD is None:
        import sys
        from torch.serialization import (INT_SIZE, LONG_SIZE, MAGIC_NUMBER, PROTOCOL_VERSION, SHORT_SIZE)
        sys_info = {"protocol_version": PROTOCOL_VERSION, "little_endian": sys.byteorder == "little",
                    "type_sizes": {"short": SHORT_SIZE, "int": INT_SIZE, "long": LONG_SIZE}}
        _HEAD = b"".join(pickle.dumps(o, protocol=2) for o in (MAGIC_NUMBER, PROTOCOL_VERSION, sys_info))
    return _HEAD


def _keys_pickle(keys: List[str], pad: int) -> bytes:
    """``pickle.dumps(keys)`` with ``pad`` (0 or >= 5) extra bytes that every unpickler - including torch's restricted
    ``weights_only`` one, which knows no ``POP`` - skips over: a junk string pushed *below* the list (``BINUNICODE``),
    which ``STOP`` leaves on the stack when it pops the result."""
    body = pickle.dumps(list(keys), protocol=2)
    assert body[:2] == b"\x80\x02" and (pad == 0 or pad >= 5)
    junk = b"" if pad == 0 else b"X" + (pad - 5).to_bytes(4, "little") + b" " * (pad - 5)
    return body[:2] + junk + body[2:]


def legacy_layout(state: Any, data_start: Optional[int] = None) -> Tuple[Layout, bytes]:
    """Layout + prefix bytes of ``state`` in the legacy ``torch.save`` container. With ``data_start`` (a previous
    layout of the same structure) the prefix is padded to end exactly there; raises ``ValueError`` if it cannot."""
    main, groups = _main_pickle(state)
    head = _head_pickles()
    keys = [ref.key for ref, _ in groups]
    bare = len(head) + len(main) + len(_keys_pickle(keys, 0))
    if data_start is None:
        data_start = (bare + _SLACK + 63) // 64 * 64
    pad = data_start - bare
    if pad < 0 or 0 < pad < 5:
        raise ValueError("prefix outgrew its slack")
    prefix = head + main + _keys_pickle(keys, pad)
    assert len(prefix) == data_start
    off = data_start
    segments, headers = [], []
    for ref, members in groups:
        esz = torch.empty(0, dtype=ref.dtype).element_size()
        numel = members[-1][1] + members[-1][0].numel() if members else 0
        headers.append((off, numel))
        base = off + 8
        for t, eoff in members:
            segments.append(_Segment(t, base + eoff * esz, t.numel() * esz))
        off = base + numel * esz
    return Layout(_signature(state), data_start, segments, off, headers), prefix


# ===================================================================================================== mappings
def _is_memory_fs(path: str) -> bool:
    """tmpfs / ramfs: no page cache write-back to miss the device's DMA writes."""
    probe = os.path.abspath(path)
    best, kind = "", ""
    try:
        with open("/proc/mounts") as f:
            for line in f:
                parts = line.split()
                if len(parts) >= 3 and (probe == parts[1] or probe.startswith(parts[1].rstrip("/") + "/")) \
                        and len(parts[1]) >= len(best):
                    best, kind = parts[1], parts[2]
    except OSError:
        return False
    return kind in ("tmpfs", "ramfs", "devtmpfs")


class MappedFile:
    """A checkpoint file mapped into the address space (and page-locked for the device when ``cuda``)."""

    def __init__(self, path: str, size: int, cuda: bool):
        self.path, self.size = path, int(size)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        tmp = f"{path}.map{os.getpid()}"
        fd = os.open(tmp, os.O_RDWR | os.O_CREAT | os.O_TRUNC, 0o644)
        try:
            os.ftruncate(fd, self.size)
            self.mm = mmap.mmap(fd, self.size, mmap.MAP_SHARED, mmap.PROT_READ | mmap.PROT_WRITE)
        finally:
            os.close(fd)
        os.replace(tmp, path)
        self.view = torch.frombuffer(self.mm, dtype=torch.uint8)
        self.ptr = self.view.data_ptr()
        self.registered = False
        if cuda:
            rc = torch.cuda.cudart().cudaHostRegister(self.ptr, self.size, 0)
            self.registered = int(rc) == 0
            if not self.registered:
                raise RuntimeError(f"cudaHostRegister failed for {path} ({self.size} bytes): {rc}")
        self.layout: Optional[Layout] = None
        self.last_event = None
        self.stage: Optional[torch.Tensor] = None        # device image of the data region [data_start, size)
        self.stage_views: Optional[list] = None          # per segment: typed device view into ``stage`` (or None)
        self.prefix_key = None                           # scalars of the object graph the current prefix was made for
        self.stage_sig = None
        self.plan_token = None                           # PersistentState binding the cached layout was made for
        self.plan_dev = None
        self.stage_runs: List[Tuple[int, int]] = []      # (file offset, bytes) of the DMA runs
        self.static_done: Dict[int, Any] = {}            # segment index -> version of a static tensor already in the image

    def rename(self, new_path: str) -> None:
        os.makedirs(os.path.dirname(new_path), exist_ok=True)
        os.replace(self.path, new_path)
        self.path = new_path

    def close(self) -> None:
        if self.registered:
            torch.cuda.cudart().cudaHostUnregister(self.ptr)
            self.registered = False
        self.view = None
        try:
            self.mm.close()
        except (BufferError, ValueError):
            pass


# ===================================================================================================== the store
class MappedCheckpointStore(CheckpointStore):
    """Drop-in :class:`CheckpointStore` whose files are persistent CUDA-registered mappings (see module docstring)."""

    def __init__(self, root: str, asynchronous: bool = True, enabled: bool = True, workers: int = 12,
                 arena_bytes: int = 8 << 30, payload_ring: int = 0, force_mapped: bool = False):
        super().__init__(root, asynchronous=asynchronous, enabled=enabled, workers=workers, arena_bytes=arena_bytes)
        self.payload_ring = int(payload_ring)
        self.mapped = bool(enabled and (force_mapped or _is_memory_fs(root if os.path.exists(root)
                                                                        else os.path.dirname(root) or "/")))
        self._files: Dict[str, MappedFile] = {}                                  # path -> mapping (stable names)
        self._ring: Dict[Tuple[str, Any], collections.deque] = {}                # (actor, signature) -> mappings
        self._ex_layouts: Dict[str, Any] = {}
        self._ring_layouts: Dict[Any, Any] = {}                                  # ring key -> (layout, prefix, scalars)
        self._graveyard: List[MappedFile] = []                                   # retired mappings, closed at close()
        self._grown: set = set()
        self._mlock = threading.RLock()
        self._lib = None
        self.dma_bytes = 0

    # ------------------------------------------------------------------ helpers
    def _native(self):
        if self._lib is None:
            from ..ops import native
            self._lib = native.load()
        return self._lib

    @staticmethod
    def _find_device(state: Any) -> Optional[torch.device]:
        stack = [state]
        while stack:
            o = stack.pop()
            if isinstance(o, torch.Tensor):
                if o.is_cuda:
                    return o.device
            elif isinstance(o, dict):
                stack.extend(o.values())
            elif isinstance(o, (list, tuple)):
                stack.extend(o)
        return None

    def _acquire(self, actor: str, path: str, layout: Layout, cuda: bool) -> MappedFile:
        """The mapping that will hold ``path``: the existing one if the layout still fits, a recycled one for
        per-round names inside a retention ring, else a new file."""
        name = os.path.basename(path)
        ringed = self.payload_ring > 0 and _PAYLOAD_NAME.match(name) is not None
        if ringed:
            key = (actor, re.sub(r"^\d+-", "", name), layout.signature)
            dq = self._ring.setdefault(key, collections.deque())
            mf = None
            if len(dq) >= self.payload_ring:
                mf = dq.popleft()
                if mf.last_event is not None:
                    mf.last_event.synchronize()
                try:
                    mf.rename(path)                 # the file of the round that left the retention window
                except OSError:                     # somebody unlinked it: its pages cannot be named again
                    self._graveyard.append(mf)
                    mf = None
            if mf is None:
                mf = MappedFile(path, layout.total, cuda)
            dq.append(mf)
            return mf
        mf = self._files.get(path)
        if mf is not None and layout.total > mf.size:
            # outgrown (FedSTIL's token memory gains one token per client and round). The old mapping is only retired:
            # cudaHostUnregister synchronises the whole device - copy stream included - so it never runs on the hot path
            self._graveyard.append(mf)
            mf = None
        if mf is None:
            grows = mf is None and path in self._grown
            self._grown.add(path)
            cap = layout.total if not grows else layout.total * 2       # a file that keeps growing gets headroom
            mf = self._files[path] = MappedFile(path, cap, cuda)
        elif mf.layout is not None and (mf.layout.signature != layout.signature):
            mf.stage = mf.stage_views = None                            # same pages, new layout: rebuild the image
        return mf

    def _write_prefix(self, mf: MappedFile, layout: Layout, prefix: bytes) -> None:
        import struct
        view = mf.view
        view[:len(prefix)] = torch.frombuffer(bytearray(prefix), dtype=torch.uint8)
        for off, numel in layout.headers:
            view[off:off + 8] = torch.frombuffer(bytearray(struct.pack("<q", numel)), dtype=torch.uint8)

    def _build_stage(self, mf: MappedFile, layout: Layout, dev: torch.device) -> None:
        """Device image of the data region (no host traffic: the per-dtype record headers in it are never transferred,
        the DMAs skip them) and one typed view per tensor."""
        ds = layout.data_start
        mf.stage = torch.empty(max(layout.total - ds, 8), dtype=torch.uint8, device=dev)
        views = []
        for seg in layout.segments:
            t = seg.tensor
            o = seg.offset - ds
            if seg.nbytes == 0 or o % t.element_size():
                views.append(None)                       # empty, or misaligned for a typed view: copied byte-wise
            else:
                views.append(mf.stage[o:o + seg.nbytes].view(t.dtype).view(t.shape))
        mf.stage_views = views
        # DMA runs: the data of each record (between two 8-byte headers)
        runs, hdrs = [], sorted(off for off, _ in layout.headers)
        for i, h in enumerate(hdrs):
            lo = h + 8
            hi = hdrs[i + 1] if i + 1 < len(hdrs) else layout.total
            if hi > lo:
                runs.append((lo, hi - lo))
        mf.stage_runs = runs

    def _issue(self, mf: MappedFile, layout: Layout, prefix: Optional[bytes], dev: Optional[torch.device]) -> None:
        """Prefix by the CPU (a few KB, only when it changed); storages through the device image + ONE DMA (CUDA) or
        by memcpy (CPU tensors)."""
        if prefix is not None:
            self._write_prefix(mf, layout, prefix)
        view = mf.view
        if dev is None:
            for seg in layout.segments:
                if seg.nbytes:
                    src = seg.tensor.detach().contiguous()
                    view[seg.offset:seg.offset + seg.nbytes] = src.reshape(-1).view(torch.uint8)
            mf.layout = layout
            return
        lib = self._native()
        from ..ops import native
        if self._copy_stream is None:
            self._copy_stream = _dedicated_stream(dev)
        cs = self._copy_stream
        cur = torch.cuda.current_stream(dev)
        if mf.last_event is not None:
            cur.wait_event(mf.last_event)                # the image is free again once its previous DMA has finished
        ds = layout.data_start
        if mf.stage is None or mf.stage_views is None or len(mf.stage_views) != len(layout.segments) \
                or mf.stage.numel() != max(layout.total - ds, 8) or mf.stage_sig != layout.signature:
            self._build_stage(mf, layout, dev)
            mf.stage_sig = layout.signature
            mf.static_done = {}
        dsts, srcs = [], []
        for i, (seg, dv) in enumerate(zip(layout.segments, mf.stage_views)):
            if not seg.nbytes:
                continue
            ver = getattr(seg.tensor, "_flpr_static", None)
            if ver is not None:                          # frozen weights: copied into the image once per version
                if mf.static_done.get(i) == ver:
                    continue
                mf.static_done[i] = ver
            src = seg.tensor.detach()
            if dv is None:
                o = seg.offset - ds
                mf.stage[o:o + seg.nbytes].copy_(src.contiguous().reshape(-1).view(torch.uint8), non_blocking=True)
            elif src.is_cuda and src.device == dev:
                dsts.append(dv)
                srcs.append(src)
            else:
                dv.copy_(src, non_blocking=True)
        if dsts:
            torch._foreach_copy_(dsts, srcs)             # the snapshot: taken here, on the producing stream
        ready = torch.cuda.Event()
        ready.record(cur)
        cs.wait_event(ready)
        base = mf.stage.data_ptr()
        for lo, nbytes in mf.stage_runs:                 # one DMA per dtype record
            rc = lib.flpr_memcpy_d2h_async(C.c_void_p(mf.ptr + lo), C.c_void_p(base + lo - ds), nbytes,
                                           C.c_void_p(cs.cuda_stream))
            native.check(rc, "flpr_memcpy_d2h_async")
            self.dma_bytes += nbytes
        ev = torch.cuda.Event()
        ev.record(cs)
        mf.last_event = ev
        mf.layout = layout
        self._last_copy_event = ev

    def fence(self, actor: Optional[str] = None) -> None:
        """Snapshots are taken into device images at ``save`` time: there is nothing for the compute stream to wait for
        (the staged parent class needs the fence because its DMAs read the live tensors)."""
        if not self.mapped:
            super().fence(actor)

    # ------------------------------------------------------------------ save
    def _save_locked(self, actor: str, state_name: str, state: Any, cover: bool, post: Optional[str]) -> None:
        if not self.mapped:
            return super()._save_locked(actor, state_name, state, cover, post)
        self._raise_pending()
        path = self.path(actor, state_name)
        if cover is False and os.path.exists(path):
            raise ValueError(f"State checkpoint has already exist in '{path}'.")
        dev = self._find_device(state)
        register = torch.cuda.is_available() and (dev is not None or self.asynchronous)
        if post == "expand_examplars":
            if self._save_examplars(actor, path, state, dev):
                return
            return super()._save_locked(actor, state_name, state, cover, post)
        if post is not None or _has_foreign(state):
            return super()._save_locked(actor, state_name, state, cover, post)
        with self._mlock:
            old = self._files.get(path)
            tok = getattr(state, "plan_token", None)
            if tok is not None and old is not None and old.layout is not None and old.plan_token == tok \
                    and old.plan_dev == dev:
                # persistent state: same structure, same tensor objects - the cached copy plan is still valid
                self._issue(old, old.layout, None, dev)
                if old.last_event is not None:
                    self._actor_events[actor] = old.last_event
                self.bytes_written += old.layout.total
                return
            if tok is not None:
                state = dict(state)             # a plain dict in the file: readers must not need our classes
            sig = _signature(state)
            scal = _scalars(state)
            if old is not None and old.layout is not None and old.layout.signature == sig and old.prefix_key == scal \
                    and not (self.payload_ring > 0 and _PAYLOAD_NAME.match(os.path.basename(path))):
                # same structure, same scalars: the pickles in the file are still right - re-point the segments only
                try:
                    layout = _rebind(old.layout, state)
                except ValueError:
                    layout = None
            else:
                layout = None
            ring_key = None
            if layout is None and self.payload_ring > 0 and _PAYLOAD_NAME.match(os.path.basename(path)):
                # per-round names: the layout (and, without changing scalars, the prefix) of last round's file of the
                # same kind is reused - nothing is pickled for an S2C payload, whose state holds tensors only
                ring_key = (actor, re.sub(r"^\d+-", "", os.path.basename(path)), sig)
                hit = self._ring_layouts.get(ring_key)
                if hit is not None and hit[2] == scal:
                    try:
                        layout = _rebind(hit[0], state)
                    except ValueError:
                        layout = None
                    if layout is not None:
                        mf = self._acquire(actor, path, layout, register)
                        self._issue(mf, layout, hit[1] if mf.prefix_key != (sig, scal) else None, dev)
                        mf.prefix_key = (sig, scal)
                        mf.plan_token, mf.plan_dev = None, dev
                        if mf.last_event is not None:
                            self._actor_events[actor] = mf.last_event
                        self.bytes_written += layout.total
                        return
            if layout is not None:
                self._issue(old, layout, None, dev)
                mf = old
            else:
                start = old.layout.data_start if (old is not None and old.layout is not None
                                                  and old.layout.signature == sig) else None
                if start is None and ring_key is not None and ring_key in self._ring_layouts:
                    start = self._ring_layouts[ring_key][0].data_start      # recycled mappings keep their data offset
                try:
                    layout, prefix = legacy_layout(state, start)
                except ValueError:
                    layout, prefix = legacy_layout(state, None)
                if ring_key is not None:
                    self._ring_layouts[ring_key] = (layout, prefix, scal)
                mf = self._acquire(actor, path, layout, register)
                if mf.layout is not None and mf.layout.signature == sig and mf.layout.data_start != layout.data_start:
                    try:
                        layout, prefix = legacy_layout(state, mf.layout.data_start)     # recycled ring mapping
                    except ValueError:
                        pass
                self._issue(mf, layout, prefix, dev)
                mf.prefix_key = scal if ring_key is None else (sig, scal)
            mf.plan_token, mf.plan_dev = tok, dev
            if mf.last_event is not None:
                self._actor_events[actor] = mf.last_event
            self.bytes_written += layout.total

    # ------------------------------------------------------------------ FedSTIL exemplar file (numpy schema)
    def _save_examplars(self, actor: str, path: str, state: Any, dev: Optional[torch.device]) -> bool:
        """``{np.int64 pid: [(ndarray fp32 prototype, class_id), ...]}`` laid out once per exemplar-set structure; the
        prototypes are cast to fp32 on the device and DMA-ed to their array offsets. Returns False to fall back."""
        import numpy as np
        if not isinstance(state, dict) or "_compact_gens" not in state:
            return False
        gens = state["_compact_gens"]
        # person / class ids are embedded in the pickle as Python ints: ONE device -> host read for all generations
        flat = [t for g in gens for t in (g["pids"].reshape(-1), g["cls"][:, :int(g["k"])].reshape(-1))]
        host = torch.cat(flat).tolist() if flat else []
        sig_parts, cur = [], 0
        host_gens = []
        for g in gens:
            P, k = int(g["pids"].numel()), int(g["k"])
            pids = host[cur:cur + P]
            cur += P
            cls = [host[cur + i * k:cur + (i + 1) * k] for i in range(P)]
            cur += P * k
            host_gens.append((pids, cls))
            sig_parts.append((tuple(pids), k, tuple(g["bank"].shape[2:]), tuple(map(tuple, cls))))
        sig = tuple(sig_parts)
        with self._mlock:
            cached = self._ex_layouts.get(path)
            if cached is None or cached[0] != sig:
                # lay the pickle out with marker-filled placeholder arrays and record every array's data offset
                out, order = {}, []
                marker = 1
                for gi, g in enumerate(gens):
                    k = int(g["k"])
                    shape = tuple(g["bank"].shape[2:])
                    pids_h, cls = host_gens[gi]
                    for pi, pid in enumerate(pids_h):
                        items = []
                        for j in range(k):
                            arr = np.full(shape, float(marker), dtype=np.float32)
                            items.append((arr, int(cls[pi][j])))
                            order.append((gi, pi, j, marker))
                            marker += 1
                        out[np.int64(pid)] = items
                buf = io.BytesIO()
                torch.save(out, buf, _use_new_zipfile_serialization=False, pickle_protocol=5)
                raw = buf.getvalue()
                offsets, pos = [], 0
                nb = int(np.prod(gens[0]["bank"].shape[2:])) * 4 if gens else 0
                for (_, _, _, mk) in order:
                    pat = np.full(min(nb // 4, 16), float(mk), dtype=np.float32).tobytes()
                    i = raw.find(pat, pos)
                    if i < 0:
                        return False
                    offsets.append(i)
                    pos = i + nb
                old = self._files.get(path)
                if old is not None and old.size >= len(raw):
                    if old.last_event is not None:
                        old.last_event.synchronize()
                    mf = old
                    mf.stage = None
                else:
                    if old is not None:
                        self._graveyard.append(old)
                    mf = self._files[path] = MappedFile(path, len(raw), torch.cuda.is_available() and
                                                        (dev is not None or self.asynchronous))
                mf.view[:len(raw)] = torch.frombuffer(bytearray(raw), dtype=torch.uint8)
                mf.layout = Layout(sig, 0, [], len(raw), [])
                cached = self._ex_layouts[path] = (sig, offsets, order, nb)
            _, offsets, order, nb = cached
            mf = self._files[path]
            if not order:
                return True
            # (generation, pid row) runs with a constant stride between consecutive arrays -> one pitched copy each
            if dev is None:
                for (gi, pi, j, _), off in zip(order, offsets):
                    src = gens[gi]["bank"][pi, j].detach().float().contiguous().reshape(-1).view(torch.uint8)
                    mf.view[off:off + nb] = src
                self.bytes_written += mf.size
                return True
            lib = self._native()
            from ..ops import native
            if self._copy_stream is None:
                self._copy_stream = _dedicated_stream(dev)
            cs = self._copy_stream
            cur = torch.cuda.current_stream(dev)
            if mf.last_event is not None:
                cur.wait_event(mf.last_event)
            lo, hi = offsets[0], offsets[-1] + nb
            if mf.stage is None or mf.stage.numel() != hi - lo:
                # device image of the file's array region, pickle bytes between the arrays included (copied up once)
                mf.stage = mf.view[lo:hi].to(dev, non_blocking=False)
            idx = 0
            for gi, g in enumerate(gens):
                k = int(g["k"])
                P = g["bank"].shape[0]
                if k <= 0 or P == 0:
                    continue
                f32 = g["bank"][:, :k].detach().float().contiguous().view(P * k, -1)       # cast on the device
                n_arr = P * k
                offs = offsets[idx:idx + n_arr]
                pitch = offs[1] - offs[0] if n_arr > 1 else nb
                uniform = all(offs[i + 1] - offs[i] == pitch for i in range(n_arr - 1))
                base = offs[0] - lo
                if uniform and pitch >= nb:
                    region = mf.stage[base:base + (n_arr - 1) * pitch + nb]
                    dst = region.as_strided((n_arr, nb), (pitch, 1))
                    if pitch % 4 == 0 and base % 4 == 0:
                        dst.view(torch.float32).copy_(f32)
                    else:
                        dst.copy_(f32.view(torch.uint8))
                else:
                    u8 = f32.view(torch.uint8)
                    for i, off in enumerate(offs):
                        mf.stage[off - lo:off - lo + nb].copy_(u8[i])
                idx += n_arr
            ready = torch.cuda.Event()
            ready.record(cur)
            cs.wait_event(ready)
            rc = lib.flpr_memcpy_d2h_async(C.c_void_p(mf.ptr + lo), native.ptr(mf.stage), hi - lo,
                                           C.c_void_p(cs.cuda_stream))
            native.check(rc, "flpr_memcpy_d2h_async")
            self.dma_bytes += hi - lo
            ev = torch.cuda.Event()
            ev.record(cs)
            mf.last_event = ev
            self._last_copy_event = ev
            self._actor_events[actor] = ev
            self.bytes_written += mf.size
            return True

    # ------------------------------------------------------------------ synchronisation / teardown
    def flush(self) -> None:
        super().flush()
        with self._mlock:
            ev = self._last_copy_event
            if ev is not None:
                ev.synchronize()

    def close(self) -> None:
        self.flush()
        with self._mlock:
            for mf in self._graveyard:
                mf.close()
            self._graveyard.clear()
            for mf in self._files.values():
                mf.close()
            for dq in self._ring.values():
                for mf in dq:
                    mf.close()
            self._files.clear()
            self._ring.clear()
        super().close()

"""ctypes bindings for ``lib/libflpr_b200.so`` (the sm_90a kernels in ``csrc/``).

Policy: on a CUDA tensor every op in :mod:`flpr_b200.ops` goes through the native library and raises loudly if the
library is missing or a launch fails — there is no silent eager fallback on a GPU box. On CPU tensors the ops use a
plain fp32 PyTorch reference (that is what the CPU test-suite exercises).
"""
from __future__ import annotations

import ctypes as C
import os
import threading
from typing import Optional

import torch

from .. import _build  # type: ignore

_lock = threading.Lock()
_lib: Optional[C.CDLL] = None

c_void_p, c_int, c_float, c_size_t, c_ll, c_double = C.c_void_p, C.c_int, C.c_float, C.c_size_t, C.c_longlong, C.c_double


class NativeError(RuntimeError):
    pass


def lib_path() -> str:
    return _build.LIB_PATH


def available() -> bool:
    return os.path.exists(_build.LIB_PATH)


def _signatures() -> dict:
    P, I, F, Z, L, D = c_void_p, c_int, c_float, c_size_t, c_ll, c_double
    return {
        "flpr_gemm_bf16": [P, P, P, I, I, I, L, L, L, I, I, I, I, F, P, P, I, P, I, I, P, P, P],
        "flpr_conv_nhwc_bf16": [P, P, P, I, I, I, I, I, I, I, I, I, I, F, P, I, P, I, P, I, L, L, L, P],
        "flpr_conv_dgrad_nhwc_bf16": [P, P, P, I, I, I, I, I, I, I, I, I, I, I, P],
        "flpr_conv_wgrad_nhwc_bf16": [P, P, P, I, I, I, I, I, I, I, I, I, I, I, P, P],
        "flpr_symm_alloc": [C.POINTER(P), Z],
        "flpr_symm_free": [P],
        "flpr_ipc_get_handle": [P, P],
        "flpr_ipc_open_handle": [P, C.POINTER(P)],
        "flpr_ipc_close": [P],
        "flpr_enable_peer": [I, I],
        "flpr_comm_read_error": [P, C.POINTER(I)],
        "flpr_comm_set_mailbox": [P, P],
        "flpr_comm_barrier": [I, I, P, D, P],
        "flpr_comm_reduce_bcast": [I, I, P, D, I, P, P, P, P, Z, I, P],
        "flpr_comm_reduce_bcast_nvls": [I, I, P, D, I, P, P, P, I, P, F, P, P, P, Z, I, P],
        "flpr_comm_set_channel": [I],
        "flpr_comm_mix": [I, I, P, D, I, I, P, P, P, P, P, P, Z, I, P],
        "flpr_comm_curv_moments": [I, I, P, D, I, P, P, P, P, P, Z, I, P],
        "flpr_comm_gather_strided": [I, I, P, D, I, P, P, Z, I, P],
        "flpr_comm_pull_copy": [I, I, P, D, P, P, P, Z, I, P],
        "flpr_fused_opt": [I, P, P, P, P, P, P, P, P, P, Z, F, F, F, F, F, I, F, F, F, F, I, P, P, P, P, P, P],
        "flpr_importance_accum": [P, P, Z, F, I, P],
        "flpr_cast_bf16": [P, P, Z, P],
        "flpr_compose": [P, P, F, P, P, Z, P],
        "flpr_ce_label_smooth": [P, P, P, P, P, I, I, L, F, F, I, I, P],
        "flpr_bn_fwd": [P, P, P, P, P, P, P, P, P, P, P, P, I, I, F, F, I, P, I, P],
        "flpr_affine_act": [P, P, P, P, P, I, I, I, P],
        "flpr_bn_bwd": [P, P, P, P, P, P, P, P, P, P, P, I, I, I, I, P],
        "flpr_bn_partials_floats": [I, I],
        "flpr_gap_fwd": [P, P, P, I, I, I, P],
        "flpr_gap_bwd": [P, P, I, I, I, P],
        "flpr_rank_eval": [P, P, P, P, P, I, I, L, P],
        "flpr_rr_sqnorm": [P, P, I, I, L, P],
        "flpr_rr_distance": [P, P, I, L, P],
        "flpr_rr_topk": [P, P, I, I, L, P],
        "flpr_rr_encode": [P, P, P, P, P, I, I, I, I, L, P],
        "flpr_rr_expand": [P, P, P, P, P, P, P, I, I, I, I, I, P],
        "flpr_rr_index": [P, P, P, I, I, I, I, P, P, P, P, P],
        "flpr_rr_jaccard": [P, P, P, I, P, P, P, P, L, P, I, I, I, F, P],
        "flpr_augment_u8": [P, P, P, I, I, I, P, P, F, F, F, F, F, F, I, P],
        "flpr_herding": [P, P, P, P, I, I, I, I, P],
        "flpr_window_attn_fwd": [P, P, P, I, I, I, I, I, F, I, P],
        "flpr_window_attn_bwd": [P, P, P, P, P, I, I, I, I, I, F, I, P],
        "flpr_s2d_pad": [P, P, I, I, I, P],
        "flpr_maxpool3x3s2": [P, P, I, I, I, I, P],
        "flpr_triplet_mine_fwd": [P, L, P, P, I, I, I, P, P, P, P, P],
        "flpr_triplet_mine_bwd": [P, P, P, P, I, P, L, P, P],
        "flpr_kd_kl": [P, P, P, P, I, I, L, L, F, I, P],
        "flpr_bce_distill": [P, P, P, P, P, I, I, I, L, L, I, P],
        "flpr_memcpy_d2h_async": [P, P, Z, P],
        "flpr_memcpy2d_d2h_async": [P, Z, P, Z, Z, Z, P],
        "flpr_host_register": [P, Z],
        "flpr_host_unregister": [P],
        "flpr_stream_create": [C.POINTER(P), I],
        "flpr_stream_destroy": [P],
    }


def declare_present(lib: C.CDLL) -> None:
    """Argument types of the int-returning entry points that ``lib`` exports (a partial library: the host builds of single
    kernel sources under the SIMT emulator of ``tests/emu``)."""
    for name, argtypes in _signatures().items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            continue
        fn.argtypes = argtypes
        fn.restype = c_int
    for name, argtypes in (("flpr_window_attn_set_tc", [c_int]),):
        try:
            fn = getattr(lib, name)
        except AttributeError:
            continue
        fn.argtypes, fn.restype = argtypes, None


def _declare(lib: C.CDLL) -> None:
    I = c_int
    for name, argtypes in _signatures().items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = I
    lib.flpr_gemm_set_persistent.argtypes = [I]
    lib.flpr_gemm_set_persistent.restype = None
    lib.flpr_gemm_set_pair.argtypes = [I]
    lib.flpr_gemm_set_pair.restype = None
    for name in ("flpr_gemm_set_debug", "flpr_gemm_set_generic_epilogue"):
        getattr(lib, name).argtypes = [I]
        getattr(lib, name).restype = None
    for name in ("flpr_gemm_last_error", "flpr_comm_last_error"):
        getattr(lib, name).restype = C.c_char_p
        getattr(lib, name).argtypes = []
    lib.flpr_window_attn_set_tc.argtypes = [I]
    lib.flpr_window_attn_set_tc.restype = None
    lib.flpr_comm_set_one_shot_bytes.argtypes = [I]
    lib.flpr_comm_set_one_shot_bytes.restype = None
    for name in ("flpr_comm_flag_page_bytes", "flpr_comm_max_clients", "flpr_comm_max_local", "flpr_comm_max_ranks",
                 "flpr_comm_max_channels"):
        getattr(lib, name).restype = I
        getattr(lib, name).argtypes = []


def load(build_if_missing: bool = False) -> C.CDLL:
    """Load (once) and return the native library."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(_build.LIB_PATH):
            if build_if_missing:
                _build.build()
            else:
                raise NativeError(
                    f"native library {_build.LIB_PATH} is missing - run `python __graft_entry__.py build` "
                    "(ops on CUDA tensors never fall back to eager PyTorch)")
        lib = C.CDLL(_build.LIB_PATH, mode=C.RTLD_GLOBAL)
        _declare(lib)
        _lib = lib
    return _lib


# ---- tests only: host builds of single kernel sources under the SIMT emulator of tests/emu ---------------------------------------
_emu_libs: list = []


def use_emulated_libraries(paths) -> None:
    """Install emulated libraries (``None`` / empty: remove them). While installed, the ops that consult
    :func:`on_device` / :func:`kernels` / :func:`stream_of` send CPU tensors down their KERNEL path - same argument
    marshalling, same ``extern "C"`` entry points as on the device - instead of the PyTorch reference."""
    _emu_libs.clear()
    for path in (paths or []):
        lib = C.CDLL(path)
        declare_present(lib)
        _emu_libs.append(lib)


class _EmuDispatch:
    """``lib.flpr_xyz`` resolved over the installed emulated libraries."""

    def __getattr__(self, name):
        for lib in _emu_libs:
            if hasattr(lib, name):
                return getattr(lib, name)
        raise AttributeError(name)


def emulated(symbol: Optional[str] = None) -> bool:
    """Emulated libraries are installed (and, with ``symbol``, one of them exports it)."""
    if symbol is None:
        return bool(_emu_libs)
    return any(hasattr(lib, symbol) for lib in _emu_libs)


def kernels():
    """The object whose attributes are the ``flpr_*`` entry points: the native library, or the emulated ones."""
    return _EmuDispatch() if _emu_libs else load()


def on_device(t: torch.Tensor, symbol: Optional[str] = None) -> bool:
    """The kernel path applies to ``t``: a CUDA tensor, or any tensor while an emulated library (exporting ``symbol``)
    is installed."""
    return t.is_cuda or emulated(symbol)


def stream_of(device) -> c_void_p:
    return c_void_p(0) if _emu_libs else stream(device)


def ptr(t: Optional[torch.Tensor]) -> c_void_p:
    if t is None:
        return c_void_p(0)
    return c_void_p(t.data_ptr())


def stream(device: Optional[torch.device] = None) -> c_void_p:
    return c_void_p(torch.cuda.current_stream(device).cuda_stream)


_streams: list = []          # keeps the ExternalStream wrappers (and thereby the handles) alive for the process


def dedicated_stream(device: Optional[torch.device] = None, priority: int = 0) -> "torch.cuda.Stream":
    """A CUDA stream that no other ``torch.cuda.Stream()`` object can alias (see ``flpr_stream_create``)."""
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    lib = load()
    with torch.cuda.device(device):
        h = c_void_p()
        check(lib.flpr_stream_create(C.byref(h), int(priority)), "flpr_stream_create")
        s = torch.cuda.ExternalStream(h.value, device=device)
    _streams.append(s)
    return s


def check(rc: int, what: str) -> None:
    if rc != 0:
        lib = load()
        msg = (lib.flpr_gemm_last_error() or b"").decode() + " | " + (lib.flpr_comm_last_error() or b"").decode()
        raise NativeError(f"{what} failed with code {rc}: {msg}")


# launch counter: bench.py reports how many flpr kernels were launched inside the timed region. Per-thread counts
# summed on read. While a CUDA graph is being captured the launches that belong to the capture are those of the
# capturing thread and of the autograd engine threads (backward runs there) - everything except OTHER client threads.
_tls = threading.local()
_counters: list = []
_client_threads: set = set()
_capture = {"owner": None, "count": 0}


def _counter() -> list:
    c = getattr(_tls, "c", None)
    if c is None:
        c = _tls.c = [0]
        with _lock:
            _counters.append(c)
    return c


def register_client_thread() -> None:
    _client_threads.add(threading.get_ident())


def count_launch(n: int = 1) -> None:
    _counter()[0] += n
    owner = _capture["owner"]
    if owner is not None:
        me = threading.get_ident()
        if me == owner or me not in _client_threads:
            _capture["count"] += n


def launches() -> int:
    """Launches of all threads."""
    return sum(c[0] for c in _counters)


def capture_count_begin() -> None:
    _capture["owner"], _capture["count"] = threading.get_ident(), 0


def capture_count_end() -> int:
    n = _capture["count"]
    _capture["owner"] = None
    return n

import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _ensure_native_library() -> None:
    """``lib/libflpr_b200.so`` is git-ignored: a fresh checkout builds it before the first test needs it (``nvcc``
    cross-compiles for sm_90a without a GPU; about a minute). A current library is left alone."""
    if os.environ.get("PYTEST_XDIST_WORKER"):
        return
    try:
        from flpr_b200 import _build
        if not _build.is_current():
            _build.build(verbose=False)
    except Exception as ex:  # noqa: BLE001  (tests that need the library then fail with its own message)
        print(f"[conftest] native build failed: {ex}")


def pytest_configure(config):
    _ensure_native_library()
    config.addinivalue_line("markers", "gpu: test needs a CUDA device")
    config.addinivalue_line("markers", "multigpu: test needs >= 2 CUDA devices")


# GPU tests that can reach kernels which were written after the builder's last GPU session (``csrc/layer_ops.cu``: the
# compose kernels of FedWeIT / fedstil-atten, the dispatch-apply kernel of the FedAvg family, the Swin token / LayerNorm
# kernels; the stride-2 route). They run AFTER every other GPU test - the kernel-level numerics suite and the flagship
# FedSTIL / ResNet path first - so that under ``pytest -x`` a surprise in them cannot hide the rest of the tier.
_LATE_GPU_KEYS = ("fedweit", "fedstil-atten", "fedavg", "fedprox", "fedcurv", "swin")


def _gpu_order(item) -> int:
    if "gpu" not in item.keywords:
        return 0
    nodeid = item.nodeid.lower()
    if "test_zz_gpu_late" in nodeid:
        return 3
    if "test_gpu_e2e" in nodeid and any(k in nodeid for k in _LATE_GPU_KEYS):
        return 2
    return 1


def pytest_collection_modifyitems(config, items):
    import torch
    items.sort(key=_gpu_order)               # stable: the order inside each class is the collection order
    has_gpu = torch.cuda.is_available()
    ngpu = torch.cuda.device_count() if has_gpu else 0
    skip_gpu = pytest.mark.skip(reason="no CUDA device")
    skip_multi = pytest.mark.skip(reason="needs >= 2 CUDA devices")
    for item in items:
        if "gpu" in item.keywords and not has_gpu:
            item.add_marker(skip_gpu)
        if "multigpu" in item.keywords and ngpu < 2:
            item.add_marker(skip_multi)

"""``server_opt_kernel`` on the GPU: every rule against the float64 oracle of ``tests/test_server_opt.py`` (same
per-step bound), at small and ResNet-50 FedAvg upload sizes, on aligned views and on views one element into their
buffer; the bf16 copy; run-to-run bitwise equality; FedAvg experiments with the kernel on the path; two or more ranks."""
import os
import subprocess
import sys

import pytest
import torch

from test_server_opt import ADAM, HP, RULES, SGD1, _means, _state, check_one_step, replay_dispatches, run_experiment

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
_SIZES = {}


def resnet50_upload_numel() -> int:
    """Length of the FedAvg upload of the ResNet-50 model of ``configs/b200/experiment_fedavg_res50_2.yaml`` (the
    prefix of its parameter arena)."""
    if "r50" not in _SIZES:
        from flpr_b200.runtime.builder import parser_model
        cfg = {"name": "resnet50", "num_classes": 8000, "last_stride": 1, "neck": "bnneck",
               "fine_tuning": ["base.layer4", "classifier"]}
        a = parser_model("fedavg", cfg, DEV, {"compute_dtype": "bf16"}).arena
        _SIZES["r50"] = a.prefix_numel or a.numel
        torch.cuda.empty_cache()
    return _SIZES["r50"]


def _on_device(t, offset):
    buf = torch.full((t.numel() + offset,), float("nan"), device=DEV, dtype=t.dtype)
    view = buf[offset:]
    view.copy_(t)
    return view


def gpu_steps(rule, n, offset, mean_offset, seed=0, check=True):
    """Three kernel steps, each checked against the oracle (``check``). ``offset`` / ``mean_offset``: elements into
    their buffers of x, m, v, the bf16 copy / of the mean."""
    from flpr_b200.ops import fused as fops, native
    x, m, v, g = _state(n, seed, 0)
    means = _means(x.clone(), g, 0)
    X, M, V = (_on_device(t, offset) for t in (x, m, v))
    SH = _on_device(torch.zeros(n, dtype=torch.bfloat16), offset)
    sgd = rule == "sgd"
    for mu in means:
        MU = _on_device(mu, mean_offset)
        before = (X.cpu(), mu, M.cpu(), None if sgd else V.cpu())
        k = native.launches()
        fops.server_opt_step(rule, X, MU, M, None if sgd else V, x_bf16=SH, **HP)
        assert native.launches() - k == 1
        torch.cuda.synchronize()
        if check:
            check_one_step(rule, HP, before, (X.cpu(), M.cpu(), V.cpu()))
            assert torch.equal(SH, X.to(torch.bfloat16))
    return X, M, V, SH


_SHAPES = [(n, o, mo) for n in (1, 3, 4, 4097) for o, mo in ((0, 0), (1, 1), (0, 1))] + \
    [("r50", 0, 0), ("r50", 1, 1)]


@pytest.mark.parametrize("rule", RULES)
@pytest.mark.parametrize("n,offset,mean_offset", _SHAPES)
def test_kernel_matches_oracle(rule, n, offset, mean_offset):
    if n == "r50":
        n = resnet50_upload_numel()
    a = gpu_steps(rule, n, offset, mean_offset, seed=7)
    b = gpu_steps(rule, n, offset, mean_offset, seed=7, check=False)
    for s, t in zip(a, b):
        assert torch.equal(s, t), "two runs differ"


def test_kernel_leaves_neighbours_alone():
    """Views one element into NaN-filled buffers: the element before the view is never written."""
    from flpr_b200.ops import fused as fops
    n = 4099
    bufs = [torch.full((n + 1,), float("nan"), device=DEV) for _ in range(4)]
    x, mean, m, v = (b[1:] for b in bufs)
    x.normal_(); mean.normal_(); m.zero_(); v.zero_()
    sh = torch.full((n + 1,), float("nan"), device=DEV, dtype=torch.bfloat16)
    fops.server_opt_step("adam", x, mean, m, v, x_bf16=sh[1:], lr=0.1)
    torch.cuda.synchronize()
    for b in bufs + [sh]:
        assert torch.isnan(b[0]).item() and torch.isfinite(b[1:].float()).all()


def _gpu_factory():
    from flpr_b200.data.synthetic import synthetic_source_factory
    return synthetic_source_factory(num_ids=4, train_per_id=4, size=(64, 32))


_GPU_TASK = {"augment_opts": {"img_size": [64, 32]}, "loader_opts": {"batch_size": 8}}


class _CountSteps:
    """Wraps ``ops.fused.server_opt_step``: the launches each call added and the device it ran on."""

    def __init__(self, monkeypatch):
        from flpr_b200.ops import fused as fops, native
        self.calls = []
        inner = fops.server_opt_step

        def wrapped(rule, x, *args, **kw):
            k = native.launches()
            inner(rule, x, *args, **kw)
            self.calls.append((x.device.type, native.launches() - k))
        monkeypatch.setattr(fops, "server_opt_step", wrapped)


def test_fedavg_adam_on_gpu_matches_float64_replay(tmp_path, monkeypatch):
    steps = _CountSteps(monkeypatch)
    root, _ = run_experiment(tmp_path, server_opt=ADAM, rounds=3, n_clients=3, device=DEV, factory=_gpu_factory(),
                             **_GPU_TASK)
    assert steps.calls == [("cuda", 1)] * 3
    assert replay_dispatches(root, ADAM, 3, 3) >= 4


def test_sgd_lr1_without_momentum_is_fedavg_on_gpu(tmp_path, monkeypatch):
    """Every dispatch of the ``sgd`` run equals the plain FedAvg mean of the uploads it checkpointed (1e-6). Unlike the
    CPU test, no second (plain) run is compared: two GPU experiments with the same configuration do not reproduce each
    other's training metrics (round-1 accuracy differed between two such runs on an H100), so a cross-run comparison
    would not isolate the server step."""
    steps = _CountSteps(monkeypatch)
    root, _ = run_experiment(tmp_path, server_opt=SGD1, n_clients=2, device=DEV, factory=_gpu_factory(), **_GPU_TASK)
    assert steps.calls == [("cuda", 1)] * 3
    assert replay_dispatches(root, SGD1, 3, 2, rtol=1e-6) >= 2


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs at least two GPUs on the box")
@pytest.mark.parametrize("nvls", ["0", "1"])
def test_server_replicas_bitwise_equal_across_gpus(tmp_path, nvls):
    n = min(torch.cuda.device_count(), 8)
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dist_server_opt_check.py")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--local-addr", "127.0.0.1",
                        "--nproc-per-node", str(n), script, "cuda", nvls], capture_output=True, text=True, timeout=900,
                       env=dict(os.environ, FLPR_TMP=str(tmp_path)))
    assert r.returncode == 0 and "DIST_SERVER_OPT OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]

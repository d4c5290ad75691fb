"""``fed_reduce_robust_kernel`` on the GPU: both rules against the float64 oracle of ``tests/test_robust_agg.py`` (same
bounds) for K in {1, 2, 3, 8, 32}, at small sizes and at the ResNet-50 FedAvg upload size; run-to-run bitwise
equality; a FedAvg experiment with a Byzantine client; two or more ranks."""
import os
import subprocess
import sys

import pytest
import torch

from test_robust_agg import check_against_oracle, poison_uploads, replay_dispatches, run_experiment, special_values

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
_SIZES = {}


def resnet50_upload_numel() -> int:
    """Length of the FedAvg upload of the ResNet-50 model of ``configs/b200/experiment_fedavg_res50_2.yaml``."""
    if "r50" not in _SIZES:
        from flpr_b200.runtime.builder import parser_model
        cfg = {"name": "resnet50", "num_classes": 8000, "last_stride": 1, "neck": "bnneck",
               "fine_tuning": ["base.layer4", "classifier"]}
        a = parser_model("fedavg", cfg, DEV, {"compute_dtype": "bf16"}).arena
        _SIZES["r50"] = a.prefix_numel or a.numel
        torch.cuda.empty_cache()
    return _SIZES["r50"]


def _comm(K, n):
    from flpr_b200.parallel.comm import FedComm
    comm = FedComm(DEV, K, arena_bytes=(K + 1) * n * 4 + (64 << 20))
    assert comm.mode == "p2p" and comm.world == 1
    comm.alloc_client_buffer("up", n)
    comm.alloc_rank_buffer("glob", n)
    return comm


@pytest.mark.parametrize("K", [1, 2, 3, 8, 32])
@pytest.mark.parametrize("n", [4, 4 * 1001, "r50"])
def test_kernel_matches_oracle(K, n):
    """Small sizes: values with ties, signed zeros, infinities and NaN (oracle on the CPU; the trimmed mean is checked
    on the coordinates without infinities or NaN). ResNet-50 size: normal values (oracle in float64 on the GPU).
    Each rule runs twice; the two results are bitwise equal."""
    from flpr_b200.methods.fedbase import trim_count
    from flpr_b200.ops import native
    big = n == "r50"
    n = resnet50_upload_numel() if big else n
    comm = _comm(K, n)
    if big:
        g = torch.Generator(device=DEV).manual_seed(K)
        vals = torch.randn(K, n, device=DEV, generator=g)
    else:
        vals = special_values(K, n, K).to(DEV)
    order = list(range(K))[::-1]
    for c in range(K):
        comm.client_view("up", c).copy_(vals[c])
    ref_vals = vals[order]
    for rule, b in (("median", 0), ("trimmed_mean", 0), ("trimmed_mean", trim_count(0.2, K)),
                    ("trimmed_mean", (K - 1) // 2)):
        outs = []
        for _ in range(2):
            comm.rank_view("glob").fill_(-7.0)
            k = native.launches()
            comm.reduce_robust("up", "glob", order, rule, b)
            assert native.launches() - k == 1
            torch.cuda.synchronize()
            comm.check_errors()
            outs.append(comm.rank_view("glob").clone())
        assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), "two runs differ"
        got = outs[0]
        if rule == "median" and not big:
            check_against_oracle(got.cpu(), ref_vals.cpu(), rule, b)
            continue
        keep = torch.isfinite(ref_vals).all(0)
        if big:
            check_against_oracle(got, ref_vals, rule, b)
        else:
            check_against_oracle(got[keep].cpu(), ref_vals[:, keep].cpu(), rule, b)
    assert comm.nvls_launches == 0
    comm.close()
    del comm, vals, ref_vals
    torch.cuda.empty_cache()


def _gpu_factory():
    from flpr_b200.data.synthetic import synthetic_source_factory
    return synthetic_source_factory(num_ids=4, train_per_id=4, size=(64, 32))


_GPU_TASK = {"augment_opts": {"img_size": [64, 32]}, "loader_opts": {"batch_size": 8}}


def test_fedavg_byzantine_on_gpu_matches_float64_replay(tmp_path, monkeypatch):
    """Four clients, client-0 uploads 1e30 / NaN; the median runs as one kernel per round on the GPU, never the NVLS
    path, and every dispatch is the float64 replay of the median over the round's upload checkpoints."""
    from flpr_b200.ops import native
    from flpr_b200.parallel.comm import FedComm
    poison_uploads(monkeypatch)
    calls = []
    inner = FedComm.reduce_robust

    def counted(self, *args, **kw):
        k, nv = native.launches(), self.nvls_launches
        inner(self, *args, **kw)
        calls.append((self.mode, native.launches() - k, self.nvls_launches - nv))
    monkeypatch.setattr(FedComm, "reduce_robust", counted)
    root, _ = run_experiment(tmp_path, "fedavg", aggregator={"name": "median"}, rounds=3, n_clients=4, device=DEV,
                             factory=_gpu_factory(), **_GPU_TASK)
    assert calls == [("p2p", 1, 0)] * 3
    assert replay_dispatches(root, {"name": "median"}, 3, 4) >= 8


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs at least two GPUs on the box")
@pytest.mark.parametrize("nvls", ["0", "1"])
def test_server_replicas_bitwise_equal_across_gpus(tmp_path, nvls):
    n = min(torch.cuda.device_count(), 8)
    script = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dist_robust_agg_check.py")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--local-addr", "127.0.0.1",
                        "--nproc-per-node", str(n), script, "cuda", nvls], capture_output=True, text=True, timeout=900,
                       env=dict(os.environ, FLPR_TMP=str(tmp_path)))
    assert r.returncode == 0 and "DIST_ROBUST_AGG OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    from test_robust_agg import oracle
    got = torch.load(tmp_path / "robust_rank0.pt", weights_only=False)["x"]
    latest = {}
    for r_ in (1, 2, 3):
        for i in range(3):
            for k in range(n):
                p = tmp_path / f"r{k}" / "ckpts" / "t-fedavg" / f"client-{i}" / f"{r_}-client-{i}-server.ckpt"
                if p.exists():
                    latest[i] = torch.load(p, weights_only=False)["incremental_model_params"]
    keys = list(got)
    stack = torch.stack([torch.cat([latest[i][k].float().flatten() for k in keys]) for i in sorted(latest)])
    assert torch.equal(torch.cat([got[k] for k in keys]), oracle(stack, "median").float())

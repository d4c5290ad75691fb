"""GPU end-to-end checks: the bf16 tensor-core head agrees with the fp32 PyTorch module, a FedSTIL / FedAvg /
FedCurv experiment runs through the native collectives on one GPU, CUDA-graph replay matches eager execution."""
import copy
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import tiny_common, tiny_experiment, tiny_factory  # noqa: E402


def _cfg():
    return {"name": "resnet50", "num_classes": 8000, "last_stride": 1, "neck": "bnneck", "atten_default": 0.9,
            "lambda_l1": 1e-3, "lambda_k": 64, "fine_tuning": ["base.layer4", "classifier"]}


def test_fast_head_matches_module_forward_backward():
    from flpr_b200.runtime.builder import parser_model
    torch.manual_seed(0)
    dev = torch.device("cuda:0")
    model = parser_model("fedstil", _cfg(), dev, {"compute_dtype": "bf16"})
    net = model.net
    fast = net._fast_head
    assert fast is not None
    proto = (torch.randn(16, 1024, 16, 8, device=dev) * 0.5).contiguous(memory_format=torch.channels_last)
    tgt = torch.randint(0, 8000, (16,), device=dev)
    net.train()
    # reference: the plain nn.Module path in fp32 on a deep copy
    ref = copy.deepcopy(net).float()
    ref._fast_head = None
    for p in ref.parameters():
        p.data = p.data.clone(memory_format=torch.contiguous_format)
    rs, rf = ref.forward_head(proto.float())
    rl = torch.nn.functional.cross_entropy(rs, tgt)
    rl.backward()
    model.arena.zero_grad()
    with model.autocast():
        s, f = net.forward_head(proto.to(torch.bfloat16))
    loss = torch.nn.functional.cross_entropy(s.float(), tgt)
    loss.backward()
    assert torch.allclose(f, rf, rtol=5e-2, atol=5e-2 * rf.abs().max().item())
    assert abs(loss.item() - rl.item()) < 5e-2 * abs(rl.item())
    g_fast = model.arena.view(model.arena.grad, "classifier.weight")
    g_ref = ref.classifier.weight.grad
    cos = torch.nn.functional.cosine_similarity(g_fast.flatten(), g_ref.flatten(), dim=0).item()
    assert cos > 0.98, cos
    g_fast = model.arena.view(model.arena.grad, "base.layer4.2.conv2.weight")
    g_ref = ref.base.layer4[2].conv2.weight.grad
    cos = torch.nn.functional.cosine_similarity(g_fast.flatten(), g_ref.flatten(), dim=0).item()
    assert cos > 0.95, cos
    # batch-norm affine gradients are accumulated by the backward kernel straight into the arena slots
    for name, mod in (("base.layer4.2.bn2", ref.base.layer4[2].bn2), ("base.layer4.0.downsample.1",
                                                                       ref.base.layer4[0].downsample[1])):
        for leaf in ("weight", "bias"):
            g_fast = model.arena.view(model.arena.grad, f"{name}.{leaf}")
            g_ref = getattr(mod, leaf).grad
            cos = torch.nn.functional.cosine_similarity(g_fast.flatten(), g_ref.flatten(), dim=0).item()
            assert cos > 0.9, (name, leaf, cos)


def test_graphed_step_matches_eager():
    from flpr_b200.runtime.arena import ArenaOptimizer
    from flpr_b200.runtime.builder import parser_criterion, parser_model
    from flpr_b200.runtime.graphs import GraphedStep
    dev = torch.device("cuda:0")
    outs = []
    for use_graph in (False, True):
        torch.manual_seed(1)
        model = parser_model("fedstil", dict(_cfg(), name="resnet18"), dev, {"compute_dtype": "bf16"})
        crit = parser_criterion({"name": "cross_entropy", "num_classes": 8000, "epsilon": 0.1})[0]
        opt = ArenaOptimizer("adam", model.arena, lr=1e-3, weight_decay=1e-5)
        model.install(opt)
        model.train()
        g = torch.Generator(device="cuda").manual_seed(5)
        xs = [torch.randn(8, 256, 16, 8, device=dev, generator=g).to(torch.bfloat16).contiguous(
            memory_format=torch.channels_last) for _ in range(6)]
        ys = [torch.randint(0, 8000, (8,), device=dev, generator=g) for _ in range(6)]

        def fn(data, target):
            opt.zero_grad()
            with model.autocast():
                score, feat = model.forward_head(data)
            crit(score=score, feature=feat, target=target).backward()
            opt.step()
        step = GraphedStep(fn, warmup=2, enabled=use_graph)
        for x, y in zip(xs, ys):
            step(x, y)
        torch.cuda.synchronize()
        outs.append(model.arena.master.clone())
    diff = (outs[0] - outs[1]).abs().max().item()
    assert diff < 5e-3, diff          # split-K atomics make the two runs non-bit-identical


ALL_METHODS = ["baseline", "ewc", "mas", "icarl", "fedavg", "fedprox", "fedcurv", "fedweit", "fedstil", "fedstil-atten"]


@pytest.mark.parametrize("method", ALL_METHODS)
def test_experiment_on_gpu(tmp_path, method):
    from flpr_b200.ops import native
    from flpr_b200.runtime.experiment import ExperimentStage
    common = tiny_common(str(tmp_path), device="cuda:0")
    common["defaults"]["task_opts"]["augment_opts"]["img_size"] = [64, 32]
    common["defaults"]["task_opts"]["loader_opts"]["batch_size"] = 8
    cfg = tiny_experiment(common, method)
    before = native.launches()
    with ExperimentStage(common, [cfg], source_factory=__import__("flpr_b200.data.synthetic", fromlist=["x"])
                         .synthetic_source_factory(num_ids=4, train_per_id=4, size=(64, 32))) as stage:
        log = stage.run_experiment(cfg)
    assert native.launches() - before > 50
    data = log.records["data"]
    for client in data.values():
        for rnd, tasks in client.items():
            for vals in tasks.values():
                for k, v in vals.items():
                    assert v == v and 0.0 <= v <= 1e4, (k, v)
    root = os.path.join(common["checkpoints_dir"], cfg["exp_name"])
    assert os.path.isdir(os.path.join(root, "client-0"))


@pytest.mark.parametrize("method", ["fedstil", "fedavg"])
def test_experiment_with_concurrent_client_streams(tmp_path, method):
    """`parallel: 2` = two client threads per device, each on its own CUDA stream (reference experiment.py:206-216)."""
    from flpr_b200.runtime.experiment import ExperimentStage
    from flpr_b200.data.synthetic import synthetic_source_factory
    common = tiny_common(str(tmp_path), device="cuda:0")
    common["parallel"] = 2
    common["defaults"]["exp_opts"].update(comm_rounds=3, online_clients=4, val_interval=3)
    common["defaults"]["task_opts"]["augment_opts"]["img_size"] = [64, 32]
    common["defaults"]["task_opts"]["loader_opts"]["batch_size"] = 8
    cfg = tiny_experiment(common, method, n_clients=4)
    with ExperimentStage(common, [cfg], source_factory=synthetic_source_factory(num_ids=4, train_per_id=4,
                                                                                size=(64, 32))) as stage:
        log = stage.run_experiment(cfg)
    data = log.records["data"]
    assert len(data) == 4
    for client in data.values():
        assert set(client.keys()) >= {"1", "2", "3"} or set(client.keys()) >= {1, 2, 3}
        for tasks in client.values():
            for vals in tasks.values():
                for k, v in vals.items():
                    assert v == v and 0.0 <= v <= 1e4, (k, v)


@pytest.mark.parametrize("name,size", [("resnet50", (256, 128)), ("resnet18", (128, 64))])
def test_native_trunk_matches_library_trunk(name, size):
    """Frozen trunk on the wgmma implicit-GEMM kernels (incl. the stride-2 convolutions) vs the cuDNN path."""
    from flpr_b200.models import resnet as R
    from flpr_b200.models.frozen import FoldedTrunk
    from flpr_b200.ops import native
    torch.manual_seed(3)
    net = getattr(R, name)(num_classes=10, last_stride=1, neck="bnneck").cuda().eval()
    net.configure_split(["base.layer4", "classifier"])
    for m in net.modules():                                   # non-trivial folded BN
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.1)
            m.running_var.uniform_(0.5, 1.5)
            m.weight.data.uniform_(0.5, 1.5)
            m.bias.data.normal_(0, 0.1)
    ft = FoldedTrunk(net, torch.bfloat16, use_graphs=False)
    x = torch.randn(16, 3, *size, device="cuda")
    assert ft._native_ok(tuple(x.shape))
    before = native.launches()
    y_native = ft(x)
    assert native.launches() - before >= 10, "the native trunk path did not run"
    ft.native = False
    ft._native_cache.clear()
    y_lib = ft(x)
    assert y_native.shape == y_lib.shape
    err = (y_native.float() - y_lib.float()).abs().max().item()
    assert err <= 5e-2 * y_lib.float().abs().max().item() + 1e-3, err
    with torch.no_grad():
        ref = net.forward_trunk(x)
    err = (y_native.float() - ref.float()).abs().max().item()
    assert err <= 8e-2 * ref.abs().max().item() + 1e-3, err


def test_swin_fused_window_attention_in_model():
    """Swin-T ReID on the GPU: fused window-attention kernel vs the SDPA path, forward and gradients of the last stage."""
    from flpr_b200.models.swin import WindowAttention
    from flpr_b200.models import nets
    from flpr_b200.ops import native
    torch.manual_seed(9)
    net = nets["swin_transformer_tiny"](num_classes=50, neck="bnneck").cuda().train()
    x = torch.randn(4, 3, 256, 128, device="cuda")
    outs = []
    for fused in (True, False):
        for m in net.modules():
            if isinstance(m, WindowAttention):
                m.fused = fused
            if isinstance(m, torch.nn.Dropout):
                m.p = 0.0
        for m in net.modules():
            if hasattr(m, "p") and m.__class__.__name__ == "DropPath":
                m.p = 0.0
        net.zero_grad()
        before = native.launches()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            score, feat = net(x)
        score.float().square().mean().backward()
        if fused:
            assert native.launches() - before >= 12, "fused attention kernels did not run"
        g = net.base.layers[3].blocks[1].attn.qkv.weight.grad.detach().clone()
        outs.append((feat.detach().float(), g.float()))
    assert torch.allclose(outs[0][0], outs[1][0], rtol=5e-2, atol=5e-2 * outs[1][0].abs().max().item())
    cos = torch.nn.functional.cosine_similarity(outs[0][1].flatten(), outs[1][1].flatten(), dim=0).item()
    assert cos > 0.98, cos


def test_fedstil_swin_experiment_on_gpu(tmp_path):
    """BASELINE config 4 in miniature: FedSTIL with a Swin-T backbone (bf16, fused window attention) end to end."""
    from flpr_b200.runtime.experiment import ExperimentStage
    from flpr_b200.data.synthetic import synthetic_source_factory
    common = tiny_common(str(tmp_path), device="cuda:0")
    common["defaults"]["model_opts"] = {"name": "swin_transformer_tiny", "num_classes": 8000, "neck": "bnneck",
                                        "fine_tuning": ["base.layers.3", "classifier"]}
    common["defaults"]["task_opts"]["augment_opts"]["img_size"] = [64, 32]
    common["defaults"]["task_opts"]["loader_opts"]["batch_size"] = 8
    cfg = tiny_experiment(common, "fedstil")
    with ExperimentStage(common, [cfg], source_factory=synthetic_source_factory(num_ids=4, train_per_id=4,
                                                                                size=(64, 32))) as stage:
        log = stage.run_experiment(cfg)
    for client in log.records["data"].values():
        for tasks in client.values():
            for vals in tasks.values():
                for k, v in vals.items():
                    assert v == v and 0.0 <= v <= 1e4, (k, v)


@pytest.mark.parametrize("name,size,batch", [("resnet50", (256, 128), 16), ("resnet18", (128, 64), 8)])
def test_native_train_mode_trunk_matches_module(name, size, batch):
    """Frozen stages in TRAIN mode (what the reference's ``model.train()`` does to the whole net for every method but
    FedSTIL, ``methods/baseline.py:38``): batch-statistic BN fed by the conv epilogue's fused statistics, running-stat
    updates, strided convolutions via TMA element strides, native stem + max-pool - against the fp32 ``nn.Module``."""
    import copy as _copy
    from flpr_b200.models import resnet as R
    torch.manual_seed(4)
    net = getattr(R, name)(num_classes=10, last_stride=1, neck="bnneck").cuda()
    net.configure_split(["base.layer4", "classifier"])
    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.weight.data.uniform_(0.5, 1.5)
            m.bias.data.normal_(0, 0.1)
    ref = _copy.deepcopy(net).float()
    trunk = R.NativeTrunk(net)
    x = torch.randn(batch, 3, *size, device="cuda").contiguous(memory_format=torch.channels_last)
    assert trunk.supported(tuple(x.shape))
    net.train(), ref.train()
    from flpr_b200.ops import native
    before = native.launches()
    y = trunk(x)
    assert native.launches() - before > 25
    ref16 = _copy.deepcopy(ref)
    with torch.no_grad():
        yr = ref.base.run_stages(x, 0, net.head_start)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            y16 = ref16.base.run_stages(x, 0, net.head_start)
    assert y.shape == yr.shape

    def rel(a, b):
        return ((a.float() - b.float()).norm() / b.float().norm()).item()
    # Yardstick: PyTorch's own bf16 (autocast, cuDNN / ATen) against the fp32 module. Forty bf16 layers with batch
    # statistics on a random-init net drift by ~25 % (rel. Frobenius) at the ResNet-50 cut - the native trunk must sit
    # at that level (measured: 0.2538 vs 0.2559), and close to the bf16 module itself.
    lib_err, nat_err = rel(y16, yr), rel(y, yr)
    print(f"native-vs-fp32 {nat_err:.4f}  bf16-autocast-vs-fp32 {lib_err:.4f}")
    assert nat_err <= 1.3 * lib_err + 1e-2, (nat_err, lib_err)
    cos = torch.nn.functional.cosine_similarity(y.float().flatten(), yr.flatten(), dim=0).item()
    cos16 = torch.nn.functional.cosine_similarity(y16.float().flatten(), yr.flatten(), dim=0).item()
    assert cos >= cos16 - 2e-2, (cos, cos16)
    # running statistics were updated like nn.BatchNorm2d does (momentum 0.1, unbiased variance)
    for (n1, b1), (n2, b2) in zip(net.base.named_modules(), ref.base.named_modules()):
        if isinstance(b1, torch.nn.BatchNorm2d) and not n1.startswith("layer4"):
            if n1 in ("bn1", "layer1.0.bn1"):            # shallow: bf16 drift is negligible, the arithmetic is checked
                assert torch.allclose(b1.running_mean, b2.running_mean, rtol=0.03, atol=5e-3), n1
                assert torch.allclose(b1.running_var, b2.running_var, rtol=0.05, atol=5e-3), n1
            else:                                        # deep: same statistics up to the drift measured above
                c = torch.nn.functional.cosine_similarity(b1.running_mean, b2.running_mean, dim=0).item()
                assert c > 0.9, (n1, c)
                ratio = (b1.running_var / b2.running_var).mean().item()
                assert 0.8 < ratio < 1.25, (n1, ratio)
            assert int(b1.num_batches_tracked) == 1, n1
    # eval mode: running statistics
    net.eval(), ref.eval()
    y = trunk(x)
    with torch.no_grad():
        yr = ref.base.run_stages(x, 0, net.head_start)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            y16 = ref.base.run_stages(x, 0, net.head_start)
    assert rel(y, yr) <= 1.3 * rel(y16, yr) + 1e-2, (rel(y, yr), rel(y16, yr))


def test_fedavg_training_step_launches_no_library_conv_or_batchnorm(tmp_path):
    """BASELINE configs 3 / 5 (FedAvg-family and local continual methods train the whole net in ``model.train()``):
    a captured training step of such a method contains no cuDNN / cuBLAS / ATen batch-norm kernel any more."""
    from torch.profiler import ProfilerActivity, profile
    from flpr_b200.runtime.builder import parser_criterion, parser_model
    from flpr_b200.runtime.arena import ArenaOptimizer
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    cfg = {"name": "resnet50", "num_classes": 8000, "last_stride": 1, "neck": "bnneck",
           "fine_tuning": ["base.layer4", "classifier"]}
    model = parser_model("fedavg", cfg, dev, {"compute_dtype": "bf16"})
    crit = parser_criterion({"name": "cross_entropy", "num_classes": 8000, "epsilon": 0.1})[0]
    opt = ArenaOptimizer("adam", model.arena, lr=1e-3, weight_decay=1e-5)
    x = torch.randn(16, 3, 256, 128, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 8000, (16,), device=dev)
    model.train()

    def step():
        opt.zero_grad()
        with model.autocast():
            score, feat = model(x)
        crit(score=score, feature=feat, target=y).backward()
        opt.step()
    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages()]
    bad = [n for n in names if any(t in n.lower() for t in ("cudnn", "cutlass", "batch_norm", "implicit_gemm",
                                                             "sgemm", "gemv", "cublas", "xmma"))]
    assert not bad, bad
    assert any("wgmma" in n for n in names), names[:20]


def test_mapped_checkpoint_store_dma_into_registered_files():
    """Snapshots of device tensors as DMAs straight into CUDA-registered RAM-disk file mappings: files are plain
    ``torch.load``-able checkpoints, overwritten in place, the exemplar file keeps the numpy schema."""
    import shutil
    import tempfile
    import numpy as np
    from flpr_b200.runtime.mapped_store import MappedCheckpointStore, _is_memory_fs
    base = "/dev/shm" if os.path.isdir("/dev/shm") else tempfile.gettempdir()
    root = tempfile.mkdtemp(dir=base, prefix="flpr_mapped_")
    try:
        st = MappedCheckpointStore(root, asynchronous=True, payload_ring=2, force_mapped=not _is_memory_fs(root))
        assert st.mapped
        dev = torch.device("cuda:0")
        w = torch.randn(512, 3, 3, 256, device=dev).permute(0, 3, 1, 2)          # channels_last view, like the arena's
        state = {"train_cnt": 3, "global_weight": {"l.global_weight": w}, "bf": torch.randn(1 << 20, device=dev).bfloat16(),
                 "cpu": torch.arange(5), "e": torch.zeros(0, device=dev)}
        for rnd in range(1, 5):
            state["train_cnt"] = rnd * 1000
            w.mul_(1.5)
            st.save("client-0", "fedstil_model", state, True)
            st.fence()
            st.save("client-0", f"{rnd}-client-0-server", {"train_cnt": rnd, "incremental_sw": {"k": w}}, True)
        gens = {"_compact_gens": [{"pids": torch.tensor([5, 6, 8], device=dev),
                                   "bank": torch.randn(3, 4, 64, 16, 8, device=dev).bfloat16(),
                                   "cls": torch.tensor([[0] * 4, [1] * 4, [2] * 4], device=dev), "k": 4}]}
        st.save("client-0", "fedstil_model_examplars", gens, True, post="expand_examplars")
        assert st.dma_bytes > 4 * w.numel() * 4
        out = st.load("client-0", "fedstil_model")
        assert out["train_cnt"] == 4000 and torch.equal(out["global_weight"]["l.global_weight"], w.cpu())
        assert torch.equal(out["bf"], state["bf"].cpu()) and out["e"].numel() == 0 and out["cpu"].tolist() == [0, 1, 2, 3, 4]
        assert sorted(os.listdir(os.path.join(root, "client-0"))) == ["3-client-0-server.ckpt", "4-client-0-server.ckpt",
                                                                      "fedstil_model.ckpt", "fedstil_model_examplars.ckpt"]
        assert st.load("client-0", "4-client-0-server")["train_cnt"] == 4
        ex = st.load("client-0", "fedstil_model_examplars")
        assert np.array_equal(ex[np.int64(6)][2][0], gens["_compact_gens"][0]["bank"][1, 2].float().cpu().numpy())
        assert ex[np.int64(8)][3][1] == 2
        st.close()
    finally:
        shutil.rmtree(root, ignore_errors=True)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs at least two GPUs on the box")
def test_peer_memory_collectives_on_two_or_more_gpus():
    """One rank per GPU under torchrun: every collective of ``csrc/fedcomm.cu`` (peer loads / stores over NVLink, the
    NVLS multicast reduce when the switch offers it, a second flag channel on a side stream, three epochs) against the
    plain tensor arithmetic; prints the achieved bandwidths."""
    import subprocess
    import sys
    n = min(torch.cuda.device_count(), 8)
    n = 8 if n >= 8 else (4 if n >= 4 else 2)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--local-addr", "127.0.0.1",
                        "--nproc-per-node", str(n), os.path.join(root, "tests", "dist_comm_check.py")],
                       capture_output=True, text=True, timeout=900, env=dict(os.environ, FLPR_BW_N=str(8_000_000)))
    print(r.stdout[-2000:])
    assert r.returncode == 0 and "DIST_COMM_CHECK OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def test_swin_head_step_runs_its_linears_on_tcgen05():
    """(Name kept from the Blackwell version of the kernel.) BASELINE config 4 (FedSTIL over Swin-T, bf16): every Linear
    of the trainable stage and the classifier runs on the wgmma GEMM (forward, dgrad, wgrad into the arena slot) - no
    cuBLAS / cuBLASLt kernel in a head step - and the step agrees with the fp32 module."""
    import copy as _copy
    from torch.profiler import ProfilerActivity, profile
    from flpr_b200.models.swin import TcLinear
    from flpr_b200.runtime.builder import parser_model
    torch.manual_seed(0)
    dev = torch.device("cuda:0")
    cfg = {"name": "swin_transformer_tiny", "num_classes": 8000, "neck": "bnneck", "atten_default": 0.9,
           "lambda_l1": 1e-3, "lambda_k": 64, "drop_path_rate": 0.0, "fine_tuning": ["base.layers.3", "classifier"]}
    model = parser_model("fedstil", cfg, dev, {"compute_dtype": "bf16"})
    net = model.net
    assert isinstance(net.classifier, TcLinear) and isinstance(net.base.layers[3].blocks[0].mlp.fc1, TcLinear)
    tokens = (torch.randn(16, 49, 768, device=dev) * 0.5)
    tgt = torch.randint(0, 8000, (16,), device=dev)
    net.train()
    ref = _copy.deepcopy(net).float()
    for p in ref.parameters():
        p.data = p.data.clone()
    rs, rf = ref.forward_head(tokens)
    torch.nn.functional.cross_entropy(rs, tgt).backward()

    def step():
        model.arena.zero_grad()
        with model.autocast():
            s, f = net.forward_head(tokens.to(torch.bfloat16))
        torch.nn.functional.cross_entropy(s.float(), tgt).backward()
        return s, f
    s, f = step()
    torch.cuda.synchronize()
    assert torch.allclose(f.float(), rf, rtol=5e-2, atol=5e-2 * rf.abs().max().item())
    for name in ("classifier.weight", "base.layers.3.blocks.1.mlp.fc2.weight", "base.layers.3.blocks.0.attn.qkv.weight"):
        g_fast = model.arena.view(model.arena.grad, name)
        g_ref = dict(ref.named_parameters())[name].grad
        cos = torch.nn.functional.cosine_similarity(g_fast.flatten(), g_ref.flatten(), dim=0).item()
        assert cos > 0.97, (name, cos)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages()]
    bad = [n for n in names if any(t in n.lower() for t in ("cublas", "cutlass", "gemv", "sgemm", "xmma", "nvjet"))]
    assert not bad, bad
    assert any("wgmma" in n for n in names)

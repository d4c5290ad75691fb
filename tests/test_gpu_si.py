"""Synaptic Intelligence on the H100: ``fused_opt_kernel<*, true>`` against the float64 oracle of ``tests/test_si.py`` at
the ResNet-50 arena size, graph-replayed SI steps against eager ones, and a ResNet-50 ``si`` run whose training step
launches only the project's kernels."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import tiny_common, tiny_experiment  # noqa: E402
from test_si import KINDS, STEPS, check_against_oracle, make_inputs, oracle_steps, run_steps  # noqa: E402

CFG = {"name": "resnet50", "num_classes": 8000, "last_stride": 1, "neck": "bnneck", "lambda_penalty": 0.1,
       "si_xi": 1e-3, "fine_tuning": ["base.layer4", "classifier"]}


@pytest.fixture(scope="module")
def res50_numel():
    from flpr_b200.runtime.builder import parser_model
    model = parser_model("si", CFG, torch.device("cuda:0"), {"compute_dtype": "bf16"})
    n = model.arena.numel
    del model
    torch.cuda.empty_cache()
    return n


@pytest.mark.parametrize("variant,penalty_wd", [("adam", True), ("adam", False), ("sgd", True),
                                                ("sgd_momentum", True)])
def test_si_kernel_matches_float64_oracle_at_resnet50_size(res50_numel, variant, penalty_wd):
    from flpr_b200.ops import native
    kind, momentum = KINDS[variant]
    wd, lam2 = (1e-2, 0.5) if penalty_wd else (0.0, 0.0)
    dev = torch.device("cuda:0")
    st = make_inputs(res50_numel, seed=11, penalty=penalty_wd)
    st = {k: (None if v is None else [x.to(dev) for x in v] if isinstance(v, list) else v.to(dev))
          for k, v in st.items()}
    ref, tol = oracle_steps(kind, momentum, st, wd, lam2)
    before = native.launches()
    got = run_steps(kind, momentum, st, wd, lam2)
    plain = run_steps(kind, momentum, st, wd, lam2, with_omega=False)
    torch.cuda.synchronize()
    assert native.launches() - before == 2 * STEPS
    check_against_oracle(got, ref, tol, kind, momentum)
    for k in ("p", "m", "v"):
        assert torch.equal(got[k], plain[k]), k              # the SI instantiation steps exactly like the plain one


def test_graphed_si_steps_equal_eager_steps(res50_numel):
    """The path integral is a pointer captured once: replayed steps must reproduce eager ones bit for bit."""
    from flpr_b200.runtime.arena import ArenaOptimizer, ParamArena
    from flpr_b200.runtime.graphs import GraphedStep
    dev = torch.device("cuda:0")
    n = res50_numel
    gen = torch.Generator(device=dev).manual_seed(3)
    grads = [torch.randn(n, device=dev, generator=gen) * 1e-3 for _ in range(6)]
    p0 = torch.randn(n, device=dev, generator=gen)
    Q = torch.rand(n, device=dev, generator=gen)
    R = Q * torch.randn(n, device=dev, generator=gen)
    outs = []
    for use_graph in (False, True):
        arena = ParamArena([("w", torch.nn.Parameter(p0.clone()))], dev, shadow=True)
        opt = ArenaOptimizer("adam", arena, lr=1e-3, weight_decay=1e-5)
        opt.Q, opt.R, opt.lam2 = Q, R, 0.1
        opt.omega = torch.zeros(n, device=dev)

        def fn(g):
            arena.grad.copy_(g)
            opt.step()
        step = GraphedStep(fn, warmup=2, enabled=use_graph)
        for g in grads:
            step(g)
        torch.cuda.synchronize()
        if use_graph:
            assert step._state and next(iter(step._state.values()))["graph"] is not None
        outs.append((arena.master.clone(), opt.m.clone(), opt.v.clone(), opt.omega.clone(), arena.shadow.clone()))
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    assert torch.count_nonzero(outs[0][3]) > 0


def test_si_resnet50_training_step_launches_no_library_conv_or_batchnorm():
    """A captured-shape ResNet-50 ``si`` training step, on the second task (active penalty, path integral), contains
    no cuDNN / cuBLAS / ATen batch-norm kernel, and runs the SI instantiation of the fused optimizer."""
    from torch.profiler import ProfilerActivity, profile
    from flpr_b200.runtime.arena import ArenaOptimizer
    from flpr_b200.runtime.builder import parser_criterion, parser_model
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    model = parser_model("si", CFG, dev, {"compute_dtype": "bf16"})
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
    model.switch_task("task-0")
    model.install(opt)
    step()
    model.switch_task("task-1")
    assert torch.count_nonzero(model.F) > 0
    model.install(opt)
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
    assert any("fused_opt_kernel<true, true>" in n for n in names), [n for n in names if "opt" in n]
    assert torch.count_nonzero(model.W) > 0


def test_si_resnet50_experiment_on_gpu(tmp_path):
    from flpr_b200.data.synthetic import synthetic_source_factory
    from flpr_b200.ops import native
    from flpr_b200.runtime.experiment import ExperimentStage
    common = tiny_common(str(tmp_path), device="cuda:0")
    common["defaults"]["task_opts"]["augment_opts"]["img_size"] = [64, 32]
    common["defaults"]["task_opts"]["loader_opts"]["batch_size"] = 8
    common["defaults"]["task_opts"]["sustain_rounds"] = 1
    common["defaults"]["exp_opts"].update(comm_rounds=3, val_interval=3)
    cfg = tiny_experiment(common, "si", n_tasks=3, model_opts=dict(common["defaults"]["model_opts"], **CFG))
    before = native.launches()
    with ExperimentStage(common, [cfg], source_factory=synthetic_source_factory(num_ids=4, train_per_id=4,
                                                                                size=(64, 32))) as stage:
        log = stage.run_experiment(cfg)
    assert native.launches() - before > 50
    data = log.records["data"]
    assert set(data) == {"client-0", "client-1"}
    for client in data.values():
        assert {"1", "2", "3"} <= set(client)
        for tasks in client.values():
            for vals in tasks.values():
                for k, v in vals.items():
                    assert v == v and 0.0 <= v <= 1e4, (k, v)
    import os
    ck = torch.load(os.path.join(common["checkpoints_dir"], cfg["exp_name"], "client-0", "si_model.ckpt"),
                    weights_only=False)
    assert set(ck) == {"net_params", "params_old", "precision_matrices", "path_integral"}
    assert any(torch.count_nonzero(t) > 0 for t in ck["precision_matrices"].values())

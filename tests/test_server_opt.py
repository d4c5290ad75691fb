"""Server optimizers of the FedAvg family (``server: server_opt:``; FedAvgM, FedAdagrad, FedAdam, FedYogi).

A float64 oracle of the update rule (checked against hand-computed values), the fp32 CPU path and the kernel source
under the SIMT emulator of ``tests/emu`` against it, configuration validation, and tiny experiments: every dispatch
recomputed from the checkpoints, ``sgd`` with lr 1 and no momentum equal to plain FedAvg, unchanged checkpoint schemas,
resume, and two gloo ranks.

Error bound of one fp32 step, per element: ``|got - ref| <= 8 * 2^-24 * (|x| + |lr * m / (sqrt(v) + tau)|)`` for ``x``
and the analogous sum of the magnitudes of the terms for ``m`` and ``v``; because ``m`` can cancel, ``|m|`` in the ``x``
bound is the sum of the magnitudes of its terms (``|beta1 m| + |(1 - beta1) d|``). Each step is compared with the oracle applied
to the fp32 state the implementation had before that step, so the bound is that of one step and does not grow with
the number of steps; the hyperparameters are rounded to fp32 for the oracle, as the kernel receives them."""
import math
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from flpr_b200.runtime.experiment import ExperimentStage
from helpers import tiny_common, tiny_experiment, tiny_factory

RULES = ["sgd", "adagrad", "adam", "yogi"]
U = 2.0 ** -24
HP = {"lr": 0.05, "momentum": 0.7, "beta1": 0.9, "beta2": 0.99, "tau": 1e-3}


# ---------------------------------------------------------------------------------------------------------- oracle
def oracle_step(rule, x, mean, m, v, *, lr, momentum=0.0, beta1=0.9, beta2=0.99, tau=1e-3):
    """One step in float64 (numpy arrays). Returns ``(x, m, v, tie)``; ``tie`` marks the Yogi elements whose sign
    ``sign(v - d^2)`` an fp32 evaluation may legitimately get wrong (``v`` and ``d^2`` within rounding of each other)."""
    x, mean, m = (np.asarray(a, dtype=np.float64) for a in (x, mean, m))
    v = np.zeros_like(x) if v is None else np.asarray(v, dtype=np.float64)
    d = mean - x
    tie = np.zeros(x.shape, dtype=bool)
    if rule == "sgd":
        m = momentum * m + d
        return x + lr * m, m, v, tie
    m = beta1 * m + (1 - beta1) * d
    d2 = d * d
    if rule == "adagrad":
        v = v + d2
    elif rule == "adam":
        v = beta2 * v + (1 - beta2) * d2
    elif rule == "yogi":
        tie = np.abs(v - d2) <= 8 * U * (np.abs(v) + d2)
        v = v - (1 - beta2) * d2 * np.sign(v - d2)
    else:
        raise ValueError(rule)
    return x + lr * m / (np.sqrt(v) + tau), m, v, tie


def f32(s):
    return float(np.float32(s))


def hp32(hp):
    return {k: f32(val) for k, val in hp.items()}


def check_one_step(rule, hp, before, after):
    """``before`` = fp32 ``(x, mean, m, v)`` ahead of the step, ``after`` = fp32 ``(x, m, v)`` it produced."""
    X, MU, M, V = (None if t is None else t.double().numpy() for t in before)
    V = np.zeros_like(X) if V is None else V
    h = hp32(hp)
    rx, rm, rv, tie = oracle_step(rule, X, MU, M, V, **h)
    assert tie.mean() < 0.01, "too many Yogi sign ties for a meaningful check"
    ok = ~tie
    d = MU - X
    # (``m`` may cancel - beta1*m and (1-beta1)*d of opposite sign - so the x bound uses |beta1*m| + |(1-beta1)*d|,
    # the bound of m's own error, in place of |m|)
    if rule == "sgd":
        bm = np.abs(h["momentum"] * M) + np.abs(d)
        ux = h["lr"] * bm
    else:
        bm = np.abs(h["beta1"] * M) + np.abs((1 - h["beta1"]) * d)
        ux = h["lr"] * bm / (np.sqrt(rv) + h["tau"])
        if rule == "adam":
            bv = np.abs(h["beta2"] * V) + (1 - h["beta2"]) * d * d
        elif rule == "adagrad":
            bv = np.abs(V) + d * d
        else:
            bv = np.abs(V) + (1 - h["beta2"]) * d * d
        gv = after[2].double().numpy()
        err = np.abs(gv - rv)[ok] - 8 * U * bv[ok]
        assert (err <= 0).all(), ("v", rule, err.max())
    gx, gm = after[0].double().numpy(), after[1].double().numpy()
    err = np.abs(gx - rx)[ok] - 8 * U * (np.abs(X) + np.abs(ux))[ok]
    assert (err <= 0).all(), ("x", rule, err.max())
    err = np.abs(gm - rm)[ok] - 8 * U * bm[ok]
    assert (err <= 0).all(), ("m", rule, err.max())


def test_oracle_matches_hand_computed_values():
    """lr 0.5, momentum 0.5, beta1 0.5, beta2 0.75, tau 1; x0 = 1 and the pseudo-gradient d = mean - x is 2 in the
    first step; the second step's mean is chosen to give the d listed per column."""
    hp = {"lr": 0.5, "momentum": 0.5, "beta1": 0.5, "beta2": 0.75, "tau": 1.0}

    def two_steps(rule, d2):
        x, m, v = np.array([1.0]), np.array([0.0]), np.array([0.0])
        x1, m1, v1, _ = oracle_step(rule, x, x + 2.0, m, v, **hp)
        x2, m2, v2, _ = oracle_step(rule, x1, x1 + d2, m1, v1, **hp)
        return [float(a[0]) for a in (x1, m1, v1, x2, m2, v2)]

    # sgd: m = 0.5*0 + 2 = 2, x = 1 + 0.5*2 = 2; then d = 1: m = 0.5*2 + 1 = 2, x = 2 + 1 = 3
    assert two_steps("sgd", 1.0) == pytest.approx([2.0, 2.0, 0.0, 3.0, 2.0, 0.0], abs=1e-15)
    # adagrad: m = 1, v = 4, x = 1 + 0.5/(2+1); then d = 1: m = 0.5 + 0.5 = 1, v = 4 + 1 = 5 (accumulates)
    assert two_steps("adagrad", 1.0) == pytest.approx(
        [1 + 0.5 / 3, 1.0, 4.0, 1 + 0.5 / 3 + 0.5 / (math.sqrt(5) + 1), 1.0, 5.0], abs=1e-15)
    # adam: m = 1, v = 0.25*4 = 1, x = 1 + 0.5/2 = 1.25; then d = 1: m = 1, v = 0.75 + 0.25 = 1, x = 1.5
    assert two_steps("adam", 1.0) == pytest.approx([1.25, 1.0, 1.0, 1.5, 1.0, 1.0], abs=1e-15)
    # yogi, v < d^2 (grows): step 1 v = 0 - 0.25*4*sign(-4) = 1, x = 1.25;
    #   d = 4: v - 16 < 0 -> v = 1 + 0.25*16 = 5, m = 0.5 + 2 = 2.5, x = 1.25 + 0.5*2.5/(sqrt 5 + 1)
    assert two_steps("yogi", 4.0) == pytest.approx(
        [1.25, 1.0, 1.0, 1.25 + 1.25 / (math.sqrt(5) + 1), 2.5, 5.0], abs=1e-15)
    # yogi, v > d^2 (shrinks): d = 0.5: v = 1 - 0.25*0.25 = 0.9375, m = 0.5 + 0.25 = 0.75
    assert two_steps("yogi", 0.5) == pytest.approx(
        [1.25, 1.0, 1.0, 1.25 + 0.375 / (math.sqrt(0.9375) + 1), 0.75, 0.9375], abs=1e-15)
    # yogi, v == d^2: sign 0, v stays
    assert two_steps("yogi", 1.0)[5] == 1.0


# ---------------------------------------------------------------------------------------------------------- fp32 steps
def _state(n, seed, offset=0):
    """fp32 ``x, m, v`` views starting ``offset`` elements into their buffers, and a generator for the means."""
    g = torch.Generator().manual_seed(seed)
    bufs = [torch.randn(n + offset, generator=g) * 0.5, torch.zeros(n + offset), torch.zeros(n + offset)]
    x, m, v = (b[offset:] for b in bufs)
    return x, m, v, g


def _means(x, g, offset):
    """Targets of three steps: close to x, far from x, and identical to x in a few elements."""
    out = []
    for k, scale in enumerate((0.01, 1.0, 0.003)):
        buf = torch.empty(x.numel() + offset)
        mu = buf[offset:]
        mu.copy_(x + scale * torch.randn(x.numel(), generator=g))
        if k == 2:
            mu[::7] = x[::7]
        out.append(mu)
    return out


def run_steps(rule, n, offset, seed=0, shadow=True):
    """Three steps of ``server_opt_step`` (whatever path is installed), each checked against the oracle; returns the
    final state."""
    from flpr_b200.ops import fused as fops
    x, m, v, g = _state(n, seed, offset)
    sh = torch.zeros(n + offset, dtype=torch.bfloat16)[offset:] if shadow else None
    for mu in _means(x.clone(), g, offset):
        before = (x.clone(), mu.clone(), m.clone(), None if rule == "sgd" else v.clone())
        fops.server_opt_step(rule, x, mu, m, None if rule == "sgd" else v, x_bf16=sh, **HP)
        check_one_step(rule, HP, before, (x, m, v))
        if sh is not None:
            assert torch.equal(sh, x.to(torch.bfloat16))
    return x, m, v


@pytest.mark.parametrize("rule", RULES)
def test_cpu_path_matches_oracle(rule):
    x, m, v = run_steps(rule, 4097, 0)
    assert torch.isfinite(x).all() and (m != 0).any()


# ---------------------------------------------------------------------------------------------------------- emulated kernel
@pytest.fixture(scope="module")
def emu_fused():
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    from emu.build_emu import build
    try:
        return build("fused_ops.cu")
    except RuntimeError as ex:
        pytest.skip(f"emulator build unavailable: {ex}")


@pytest.mark.parametrize("rule", RULES)
@pytest.mark.parametrize("n", [1, 3, 4, 4097])
@pytest.mark.parametrize("offset", [0, 1])
def test_emulated_kernel_matches_oracle(emu_fused, rule, n, offset):
    """``server_opt_kernel`` itself, run on the CPU: the vector path (aligned views) with its scalar tail, and the scalar
    path (views one element into their buffer)."""
    from flpr_b200.ops import fused as fops, native
    fops.use_emulated_libraries([emu_fused])
    try:
        before = native.launches()
        run_steps(rule, n, offset, seed=n + offset)
        assert native.launches() - before == 3, "the emulated kernel did not run"
    finally:
        fops.use_emulated_libraries(None)


def test_emulated_kernel_rejects_bad_rule_and_missing_state(emu_fused):
    import ctypes as C
    from flpr_b200.ops import fused as fops, native
    fops.use_emulated_libraries([emu_fused])
    try:
        lib = native.kernels()
        x, mu, m, v = (torch.zeros(8) for _ in range(4))
        P = native.ptr
        call = lambda rule, mm, vv: lib.flpr_server_opt(rule, P(x), P(mu), P(mm), P(vv), P(None), 8, 1.0, 0.0, 0.9,
                                                        0.99, 1e-3, C.c_void_p(0))
        assert call(4, m, v) == -2 and call(-1, m, v) == -2
        assert call(2, None, v) == -3 and call(3, m, None) == -3 and call(1, m, None) == -3
        assert call(0, m, None) == 0 and call(2, m, v) == 0
    finally:
        fops.use_emulated_libraries(None)


# ---------------------------------------------------------------------------------------------------------- validation
@pytest.mark.parametrize("bad", [
    {"name": "rmsprop", "lr": 0.1}, {"lr": 0.1}, {"name": "adam", "lr": 0.1, "eps": 1e-8},
    {"name": "sgd", "lr": 0.1, "beta1": 0.9}, {"name": "adam"}, {"name": "adam", "lr": 0.0},
    {"name": "sgd", "lr": -1.0}, {"name": "yogi", "lr": float("nan")}, {"name": "sgd", "lr": 1.0, "momentum": 1.0},
    {"name": "sgd", "lr": 1.0, "momentum": -0.1}, {"name": "adam", "lr": 1.0, "beta1": 1.0},
    {"name": "adagrad", "lr": 1.0, "beta1": -0.5}, {"name": "yogi", "lr": 1.0, "beta2": 1.0},
    {"name": "adam", "lr": 1.0, "beta2": 1.5}, {"name": "adam", "lr": 1.0, "tau": 0.0},
    {"name": "yogi", "lr": 1.0, "tau": -1e-3}, "adam"])
def test_bad_server_opt_is_refused(bad):
    from flpr_b200.methods.fedbase import parse_server_opt
    with pytest.raises(ValueError):
        parse_server_opt(bad)


def test_server_opt_defaults():
    from flpr_b200.methods.fedbase import parse_server_opt
    assert parse_server_opt(None) is None
    assert parse_server_opt({"name": "sgd", "lr": 1}) == {"name": "sgd", "lr": 1.0, "momentum": 0.0}
    assert parse_server_opt({"name": "adagrad", "lr": 0.1}) == {"name": "adagrad", "lr": 0.1, "beta1": 0.9,
                                                                 "beta2": 0.99, "tau": 1e-3}


def test_bad_server_opt_fails_at_server_construction(tmp_path):
    from flpr_b200.runtime.builder import parser_server
    common = tiny_common(str(tmp_path))
    cfg = tiny_experiment(common, "fedcurv")
    cfg["server"]["server_opt"] = {"name": "adam", "lr": 0.01, "tau": 0}
    with pytest.raises(ValueError, match="tau"):
        parser_server(cfg, common)


@pytest.mark.parametrize("method", ["fedstil", "fedstil-atten", "fedweit", "ewc", "mas", "icarl", "baseline"])
def test_server_opt_refused_for_methods_without_a_fedavg_server(tmp_path, method):
    from flpr_b200.runtime.builder import parser_server
    common = tiny_common(str(tmp_path))
    cfg = tiny_experiment(common, method)
    cfg["server"]["server_opt"] = {"name": "adam", "lr": 0.01}
    with pytest.raises(ValueError, match=method):
        parser_server(cfg, common)


# ---------------------------------------------------------------------------------------------------------- experiments
ADAM = {"name": "adam", "lr": 0.01, "beta1": 0.9, "beta2": 0.99, "tau": 1e-3}


def run_experiment(tmp, method="fedavg", server_opt=None, rounds=3, n_clients=3, device="cpu", factory=None,
                   **common_over):
    common = tiny_common(str(tmp), device=device)
    common["defaults"]["exp_opts"]["comm_rounds"] = rounds
    for key, val in common_over.items():
        common["defaults"]["task_opts"][key].update(val)
    cfg = tiny_experiment(common, method, n_clients=n_clients)
    if server_opt is not None:
        cfg["server"]["server_opt"] = dict(server_opt)
    with ExperimentStage(common, [cfg], source_factory=factory or tiny_factory()) as stage:
        log = stage.run_experiment(cfg)
    return os.path.join(common["checkpoints_dir"], cfg["exp_name"]), log


def _load(root, actor, name):
    path = os.path.join(root, actor, f"{name}.ckpt")
    return torch.load(path, weights_only=False) if os.path.exists(path) else None


def replay_dispatches(root, server_opt, rounds, n_clients, rtol=1e-5):
    """Recompute in float64 the server replica after every round from the checkpoints the run wrote, and compare it with
    every dispatch of the next round. Returns the number of dispatches compared."""
    names = [f"client-{i}" for i in range(n_clients)]
    o = dict(server_opt)
    rule = o.pop("name")
    latest, cnt = {}, {}
    m = v = None
    checked = 0
    for r in range(1, rounds):
        prev = None
        for n in names:                            # the replica before round r's step: any dispatch of round r
            st = _load(root, "server", f"{r}-server-{n}")
            if st is not None:
                prev = st.get("incremental_model_params") or st["integrated_model_params"]
                break
        for n in names:                            # uploads of round r; offline clients keep their last one
            up = _load(root, n, f"{r}-{n}-server")
            if up is not None:
                latest[n] = {k: t.double() for k, t in up["incremental_model_params"].items()}
                cnt[n] = float(up["train_cnt"])
        keys = sorted(next(iter(latest.values())))
        total = sum(cnt.values())
        x = torch.cat([prev[k].double().flatten() for k in keys]).numpy()
        mean = sum(cnt[n] * torch.cat([latest[n][k].flatten() for k in keys]) for n in latest) / total
        if m is None:
            m, v = np.zeros_like(x), np.zeros_like(x)
        x, m, v, _ = oracle_step(rule, x, mean.numpy(), m, v, **o)
        for n in names:
            st = _load(root, "server", f"{r + 1}-server-{n}")
            if st is None:
                continue
            got = st.get("incremental_model_params") or st["integrated_model_params"]
            got = torch.cat([got[k].double().flatten() for k in keys]).numpy()
            np.testing.assert_allclose(got, x, rtol=rtol, atol=1e-8, err_msg=f"round {r + 1} dispatch to {n}")
            checked += 1
    return checked


def test_fedavg_adam_dispatches_match_float64_replay(tmp_path):
    """3 clients, 2 online per round: stale uploads stay in the mean, and some dispatches are first contacts."""
    root, _ = run_experiment(tmp_path, server_opt=ADAM, rounds=3, n_clients=3)
    assert replay_dispatches(root, ADAM, 3, 3) >= 4


def _flat_metrics(log):
    out = {}
    for client, rounds in log.records["data"].items():
        for rnd, tasks in rounds.items():
            for task, vals in tasks.items():
                for k, val in vals.items():
                    if isinstance(val, (int, float)):
                        out[(client, rnd, task, k)] = float(val)
    return out


def _model_files(root):
    out = {}
    for actor in sorted(os.listdir(root)):
        d = os.path.join(root, actor)
        if actor.startswith("_") or not os.path.isdir(d):
            continue
        for name in sorted(os.listdir(d)):
            if name.endswith(".ckpt"):
                out[f"{actor}/{name}"] = torch.load(os.path.join(d, name), weights_only=False)
    return out


def _tensors(obj, prefix=""):
    if torch.is_tensor(obj):
        return {prefix: obj}
    if isinstance(obj, dict):
        out = {}
        for k, val in obj.items():
            out.update(_tensors(val, f"{prefix}/{k}"))
        return out
    return {}


SGD1 = {"name": "sgd", "lr": 1.0}


def compare_sgd1_with_fedavg(root_a, log_a, root_b, log_b):
    """``sgd`` with lr 1 and no momentum is FedAvg: ``x + (mean - x)``.

    * the logged metrics agree within 1e-6 relative;
    * the first server step's dispatch (round 2 - both runs had identical inputs up to it) agrees within 1e-6;
    * every dispatch of the ``sgd`` run equals the plain mean of the uploads it checkpointed (1e-6).
    Later weights of the two runs are not compared with each other: ``x + (mean - x)`` may differ from ``mean`` in the
    last bit, and the clients' Adam steps amplify a last-bit difference wherever a gradient is close to zero."""
    ma, mb = _flat_metrics(log_a), _flat_metrics(log_b)
    assert set(ma) == set(mb) and len(ma) > 10
    for k in ma:
        assert abs(ma[k] - mb[k]) <= 1e-6 * max(abs(ma[k]), abs(mb[k])) + 1e-12, (k, ma[k], mb[k])
    fa, fb = _model_files(root_a), _model_files(root_b)
    assert set(fa) == set(fb)
    second = [f for f in fa if f.startswith("server/2-")]
    assert second
    for f in second:
        ta, tb = _tensors(fa[f]), _tensors(fb[f])
        assert set(ta) == set(tb)
        for k in ta:
            a, b = ta[k].double(), tb[k].double()
            assert torch.allclose(a, b, rtol=1e-6, atol=1e-6 * float(a.abs().max()) + 1e-12), (f, k)
    assert replay_dispatches(root_b, SGD1, 3, 2, rtol=1e-6) >= 2


def test_sgd_lr1_without_momentum_is_fedavg(tmp_path):
    root_a, log_a = run_experiment(tmp_path / "plain", n_clients=2)
    root_b, log_b = run_experiment(tmp_path / "sgd", server_opt=SGD1, n_clients=2)
    compare_sgd1_with_fedavg(root_a, log_a, root_b, log_b)


def _key_tree(obj):
    if isinstance(obj, dict):
        return {k: _key_tree(val) for k, val in obj.items()}
    return type(obj).__name__ if not torch.is_tensor(obj) else ("tensor", tuple(obj.shape))


@pytest.mark.parametrize("method", ["fedprox", "fedcurv"])
def test_yogi_keeps_checkpoint_and_payload_schemas(tmp_path, method):
    yogi = {"name": "yogi", "lr": 0.01}
    root_a, _ = run_experiment(tmp_path / "plain", method, rounds=2, n_clients=2)
    root_b, _ = run_experiment(tmp_path / "yogi", method, server_opt=yogi, rounds=2, n_clients=2)
    fa, fb = _model_files(root_a), _model_files(root_b)
    assert set(fa) == set(fb) and any("-server-" in f for f in fa)
    for f in fa:
        assert _key_tree(fa[f]) == _key_tree(fb[f]), f
    moved = [f for f in fa if f.startswith("server/2-")]
    assert moved and any(not torch.equal(_tensors(fa[f])[k], _tensors(fb[f])[k]) for f in moved
                         for k in _tensors(fa[f])), "the server optimizer did not change the dispatch"


# ---------------------------------------------------------------------------------------------------------- resume
def _run_resumable(tmp, rounds, resume=False, interval=0, drop_moments=False):
    from flpr_b200.runtime import resume as R
    from flpr_b200.runtime.explog import ExperimentLog
    from flpr_b200.utils.misc import DeviceTimer, same_seeds
    common = tiny_common(tmp)
    common["defaults"]["exp_opts"].update(comm_rounds=rounds, val_interval=100)
    common["defaults"]["task_opts"]["sustain_rounds"] = 2
    cfg = tiny_experiment(common, "fedavg")
    cfg["server"]["server_opt"] = dict(ADAM)
    cfg["engine_opts"].update(resume=resume, resume_interval=interval, val_at_round0=False)
    with ExperimentStage(common, [cfg], source_factory=tiny_factory()) as stage:
        same_seeds(cfg["random_seed"])
        store, comm, server, clients, names = stage.build(cfg)
        log = ExperimentLog(os.path.join(tmp, "log.json"), enabled=False)
        timer = DeviceTimer(stage.device)
        first = 1
        if resume and R.available(store, 0):
            if drop_moments:
                load = server.load_resume_extra
                server.load_resume_extra = lambda extra: load({k: val for k, val in extra.items()
                                                               if k not in ("server_opt_m", "server_opt_v")})
            first = R.load(stage, store, server, clients, comm) + 1
        for r in range(first, rounds + 1):
            stage._process_one_round(r, server, clients, names, cfg, log, timer, comm)
            if interval and r % interval == 0:
                R.save(stage, store, r, server, clients, comm)
        store.flush()
        out = {"server": server.model.arena.master.clone(), "m": server.opt_m.clone(), "v": server.opt_v.clone(),
               "clients": [c.model.arena.master.clone() for c in clients]}
        store.close()
        if comm is not None:
            comm.close()
    return out, first


def test_resume_carries_the_server_moments(tmp_path):
    full, _ = _run_resumable(str(tmp_path / "a"), 4)
    _run_resumable(str(tmp_path / "b"), 2, interval=2)
    shutil.copytree(tmp_path / "b", tmp_path / "c")
    cont, first = _run_resumable(str(tmp_path / "b"), 4, resume=True, interval=2)
    assert first == 3
    for k in ("server", "m", "v"):
        assert torch.allclose(cont[k], full[k], atol=1e-5, rtol=1e-5), k
    for a, b in zip(cont["clients"], full["clients"]):
        assert torch.allclose(a, b, atol=1e-5)
    # negative control: the same continuation without the moments in the manifest restarts them from zero
    lost, first = _run_resumable(str(tmp_path / "c"), 4, resume=True, interval=2, drop_moments=True)
    assert first == 3
    assert not torch.allclose(lost["server"], full["server"], atol=1e-5, rtol=1e-5)


def test_resume_manifest_unchanged_without_server_opt(tmp_path):
    from flpr_b200.methods.fedbase import FedServer
    server = FedServer.__new__(FedServer)
    server.server_opt = None
    assert server.resume_extra() == {}


# ---------------------------------------------------------------------------------------------------------- two ranks
def test_gloo_two_ranks_keep_identical_server_state(tmp_path):
    """World size 2 on gloo: replicas, ``m`` and ``v`` bit-identical across ranks after 3 rounds, and equal (1e-6) to the
    server step replayed in one process, in fp32, from the uploads both ranks checkpointed."""
    from flpr_b200.ops import fused as fops
    script = os.path.join(os.path.dirname(__file__), "dist_server_opt_check.py")
    env = dict(os.environ, FLPR_TMP=str(tmp_path), OMP_NUM_THREADS="2")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--local-addr", "127.0.0.1",
                        "--nproc-per-node", "2", script, "cpu"], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "DIST_SERVER_OPT OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    got = torch.load(tmp_path / "server_opt_rank0.pt", weights_only=False)
    keys, (x, m, v) = replay_world1(tmp_path, ADAM, 3, fops)
    for name, b in (("x", x), ("m", m), ("v", v)):
        a = torch.cat([got[name][k] for k in keys])
        assert torch.allclose(a, b, rtol=1e-6, atol=1e-6 * float(b.abs().max())), name


def replay_world1(base, server_opt, rounds, fops):
    """The server role of a 2-rank run replayed in one process (fp32 mean, ``server_opt_step``) from the payload
    checkpoints under ``base/r0`` and ``base/r1`` (each rank wrote its own clients' uploads)."""
    roots = [os.path.join(str(base), f"r{k}", "ckpts", "t-fedavg") for k in (0, 1)]

    def find(actor, name):
        for root in roots:
            st = _load(root, actor, name)
            if st is not None:
                return st
        return None

    o = dict(server_opt)
    rule = o.pop("name")
    names = ["client-0", "client-1"]
    latest, cnt = {}, {}
    x = m = v = None
    for r in range(1, rounds + 1):
        for n in names:
            up = find(n, f"{r}-{n}-server")
            if up is not None:
                latest[n], cnt[n] = up["incremental_model_params"], float(up["train_cnt"])
        keys = list(next(iter(latest.values())))
        if x is None:
            st = find("server", f"1-server-{names[0]}") or find("server", f"1-server-{names[1]}")
            init = st["integrated_model_params"]
            x = torch.cat([init[k].float().flatten() for k in keys])
            m, v = torch.zeros_like(x), torch.zeros_like(x)
        order = sorted(latest)
        stack = torch.stack([torch.cat([latest[n][k].float().flatten() for k in keys]) for n in order])
        w = torch.tensor([cnt[n] for n in order], dtype=torch.float32)
        mean = ((w / w.sum())[:, None] * stack).sum(0)
        fops.server_opt_step(rule, x, mean, m, v, **o)
    return keys, (x, m, v)

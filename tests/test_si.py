"""Synaptic Intelligence (``methods/si.py``; Zenke, Poole and Ganguli, ICML 2017): the path integral accumulated by the
fused optimizer step (CPU twin and ``fused_opt_kernel<*, true>`` under the SIMT emulator of ``tests/emu``) against a
float64 oracle, the path-integral property on a separable quadratic, consolidation at task switches, the penalty
gradient against autograd, and tiny end-to-end / resume runs."""
import math
import os
import shutil

import pytest
import torch
import torch.nn as nn

from helpers import tiny_common, tiny_experiment, tiny_factory

# Per-element bound of the fp32 step against the float64 oracle, accumulated over the steps. Every fp32 result may carry
# ULP8 = 8 fp32 ulps of relative error per step (a handful of roundings per formula). On top of that the kernel gets its
# hyper-parameters in fp32: 1 - beta and the bias corrections 1 - beta^t lose their leading bits to cancellation, a
# relative error of up to HP_ERR = 4 ulps * (1/(1-b1) + 1/(1-b2) + 1/(1-b1^t) + 1/(1-b2^t)) on an Adam update / moment.
# With dp = p_t+1 - p_t:
#   err(dp) = ULP8 * (|p_t| + |p_t+1| + |dp|) + HP_ERR * |dp|                  (a difference of two rounded weights)
#   |p32 - p64| <= sum_t err(dp)
#   |W32 - W64| <= sum_t ULP8 * |W_t+1| + |g_t| * err(dp)                         (W += -g * dp)
#   |m32 - m64| <= sum_t (ULP8 + HP_ERR) * |m_t+1| + k * |p32 - p64|,  |v32 - v64| likewise with 2 |grad| k
# where k = wd + 2 lam2 |Q| carries the weight error into the penalty / weight-decay gradient.
ULP8 = 8 * 2.0 ** -24
STEPS = 4
KINDS = {"adam": ("adam", 0.0), "sgd": ("sgd", 0.0), "sgd_momentum": ("sgd", 0.9)}
HP = dict(lr=1e-2, beta1=0.9, beta2=0.999, eps=1e-8)


def make_inputs(n, seed, penalty):
    g = torch.Generator().manual_seed(seed)
    r = lambda scale=1.0: torch.randn(n, generator=g) * scale  # noqa: E731
    st = {"p": r(), "m": r(0.01), "v": r(0.01).abs(), "W": r(1e-3),
          "gs": [r(0.1) for _ in range(STEPS)]}
    st["Q"], st["R"] = (r().abs(), r()) if penalty else (None, None)
    return st


def oracle_steps(kind, momentum, st, wd, lam2):
    """float64 reference of STEPS SI steps (optimizer update, then ``W += -g * (p_new - p_old)`` with the loss
    gradient ``g``); returns the final state and the per-element error bounds of the fp32 implementations."""
    d = lambda t: None if t is None else t.double()  # noqa: E731
    p, m, v, W, Q, R = (d(st[k]) for k in ("p", "m", "v", "W", "Q", "R"))
    tol = {k: torch.zeros_like(p) for k in ("p", "m", "v", "W")}
    k_pen = wd + (2 * lam2 * Q.abs() if Q is not None else 0.0)
    b1, b2 = HP["beta1"], HP["beta2"]
    for t, g in enumerate(st["gs"], start=1):
        g = g.double()
        grad = g + wd * p
        if Q is not None:
            grad = grad + 2 * lam2 * (Q * p - R)
        hp_err = 0.0
        if kind == "adam":
            hp_err = 4 * 2.0 ** -24 * (1 / (1 - b1) + 1 / (1 - b2) + 1 / (1 - b1 ** t) + 1 / (1 - b2 ** t))
            m = b1 * m + (1 - b1) * grad
            v = b2 * v + (1 - b2) * grad * grad
            np_ = p - HP["lr"] / (1 - b1 ** t) * m / (v.sqrt() / math.sqrt(1 - b2 ** t) + HP["eps"])
        else:
            step = grad
            if momentum:
                m = momentum * m + grad
                step = m
            np_ = p - HP["lr"] * step
        dp = np_ - p
        W = W - g * dp
        err_dp = ULP8 * (p.abs() + np_.abs() + dp.abs()) + hp_err * dp.abs()
        tol["p"] += err_dp
        tol["W"] += ULP8 * W.abs() + g.abs() * err_dp
        tol["m"] += (ULP8 + hp_err) * m.abs() + k_pen * tol["p"]
        tol["v"] += (ULP8 + hp_err) * v.abs() + 2 * grad.abs() * k_pen * tol["p"]
        p = np_
    return {"p": p, "m": m, "v": v, "W": W}, tol


def run_steps(kind, momentum, st, wd, lam2, with_omega=True, pass_none=True):
    from flpr_b200.ops import fused as fops
    p, m, v, W = (st[k].clone() for k in ("p", "m", "v", "W"))
    for t, g in enumerate(st["gs"], start=1):
        kw = {}
        if with_omega:
            kw["omega"] = W
        elif pass_none:
            kw["omega"] = None
        fops.fused_optimizer_step(kind, p, g.clone(), m if (kind == "adam" or momentum) else None,
                                  v if kind == "adam" else None, lr=HP["lr"], step=t, beta1=HP["beta1"],
                                  beta2=HP["beta2"], eps=HP["eps"], weight_decay=wd, momentum=momentum,
                                  Q=st["Q"], R=st["R"], lam2=lam2, **kw)
    return {"p": p, "m": m, "v": v, "W": W}


@pytest.fixture(scope="module")
def emu_paths():
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    from emu.build_emu import build
    try:
        return [build("fused_ops.cu"), build("loss_ops.cu")]
    except RuntimeError as ex:
        pytest.skip(f"emulator build unavailable: {ex}")


def _emulated(paths):
    from flpr_b200.ops import native

    class _Ctx:
        def __enter__(self):
            native.use_emulated_libraries(paths)
            self.before = native.launches()
            return self

        def __exit__(self, *exc):
            self.launches = native.launches() - self.before
            native.use_emulated_libraries(None)
            return False
    return _Ctx()


def check_against_oracle(got, ref, tol, kind, momentum):
    keys = ["p", "W"] + (["m"] if kind == "adam" or momentum else []) + (["v"] if kind == "adam" else [])
    for k in keys:
        err = (got[k].double() - ref[k]).abs()
        bad = err > tol[k]
        assert not bad.any(), (k, float(err.max()), float((err / tol[k]).max()))


# ---------------------------------------------------------------------------------------------------- 1. step oracle
@pytest.mark.parametrize("n", [4, 8, 4100])
@pytest.mark.parametrize("penalty_wd", [False, True])
@pytest.mark.parametrize("variant", list(KINDS))
@pytest.mark.parametrize("path", ["cpu", "emulated"])
def test_si_step_matches_float64_oracle(request, path, variant, penalty_wd, n):
    kind, momentum = KINDS[variant]
    wd, lam2 = (1e-2, 0.5) if penalty_wd else (0.0, 0.0)
    st = make_inputs(n, seed=n + 7 * penalty_wd, penalty=penalty_wd)
    ref, tol = oracle_steps(kind, momentum, st, wd, lam2)
    if path == "cpu":
        got = run_steps(kind, momentum, st, wd, lam2)
        plain = run_steps(kind, momentum, st, wd, lam2, with_omega=False, pass_none=False)
        explicit = run_steps(kind, momentum, st, wd, lam2, with_omega=False, pass_none=True)
    else:
        with _emulated(request.getfixturevalue("emu_paths")) as ctx:
            got = run_steps(kind, momentum, st, wd, lam2)
            plain = run_steps(kind, momentum, st, wd, lam2, with_omega=False, pass_none=False)
            explicit = run_steps(kind, momentum, st, wd, lam2, with_omega=False, pass_none=True)
        assert ctx.launches == 3 * STEPS, "the emulated kernel did not run"
    check_against_oracle(got, ref, tol, kind, momentum)
    for k in ("p", "m", "v", "W"):
        assert torch.equal(explicit[k], plain[k]), k         # omega=None is the call without the argument
    for k in ("p", "m", "v"):
        assert torch.equal(got[k], plain[k]), k              # the path integral does not touch the step itself
    assert torch.equal(plain["W"], st["W"])


# ------------------------------------------------------------------------------------------- 2. path-integral property
@pytest.mark.parametrize("path", ["cpu", "emulated"])
def test_path_integral_of_a_separable_quadratic(request, path):
    """SGD on ``L = 1/2 sum h_k (p_k - a_k)^2``: with ``e_t = p_t - a = r^t e_0``, ``r = 1 - lr h``, the path integral is
    ``W = lr h^2 e_0^2 (1 - r^2T) / (1 - r^2)`` exactly, and ``sum W`` equals the loss drop ``L(p_0) - L(p_T)`` up to the
    factor ``1 / (1 - lr h / 2)``: a first-order error in ``lr``."""
    from flpr_b200.ops import fused as fops
    n, T, lr = 64, 200, 1e-3
    gen = torch.Generator().manual_seed(3)
    h = torch.rand(n, generator=gen) * 4 + 0.5
    a = torch.randn(n, generator=gen)
    p0 = a + torch.randn(n, generator=gen)

    def run():
        p, W = p0.clone(), torch.zeros(n)
        for t in range(1, T + 1):
            fops.fused_optimizer_step("sgd", p, h * (p - a), None, None, lr=lr, step=t, omega=W)
        return p, W
    if path == "cpu":
        p, W = run()
    else:
        with _emulated(request.getfixturevalue("emu_paths")):
            p, W = run()
    hd, ad, e0 = h.double(), a.double(), (p0 - a).double()
    r = 1 - lr * hd
    closed = lr * hd ** 2 * e0 ** 2 * (1 - r ** (2 * T)) / (1 - r ** 2)
    assert torch.allclose(W.double(), closed, rtol=1e-4, atol=1e-9), float((W.double() - closed).abs().max())
    loss = lambda q: 0.5 * (hd * (q.double() - ad) ** 2).sum()  # noqa: E731
    drop = float(loss(p0) - loss(p))
    assert drop > 0
    assert abs(float(W.double().sum()) - drop) <= lr * float(h.max()) * drop


# ------------------------------------------------------------------------------------------------- 3. consolidation
def _tiny_si(lam=0.5, xi=0.1):
    from flpr_b200.methods import si
    torch.manual_seed(0)
    return si.Model(nn.Linear(2, 2), lambda_penalty=lam, si_xi=xi).materialize("cpu")   # 4 + 2 (+ 2 pad)


def test_consolidation_over_two_task_switches():
    m = _tiny_si(xi=0.1)
    a = m.arena
    n = a.numel
    assert n == 8 and m.W.shape == (8,)
    W_id = id(m.W)
    dispatched = torch.arange(n, dtype=torch.float32) * 0.1                 # a dispatch before the first task
    a.master.copy_(dispatched)
    m.switch_task("t0")                                                       # first task: nothing to consolidate
    assert torch.count_nonzero(m.F) == 0 and torch.equal(m.p_old, dispatched) and m.task_name == "t0"
    p1 = dispatched + torch.tensor([0.5, -0.5, 0.0, 1.0, 0.2, -0.1, 0.3, 0.0])
    w1 = torch.tensor([0.2, 0.1, 0.0, -0.3, 0.05, 0.4, 0.0, 0.1])
    a.master.copy_(p1)
    m.W.copy_(w1)
    m.switch_task("t0")                                                       # next round of the same task
    assert torch.count_nonzero(m.F) == 0 and torch.equal(m.p_old, dispatched) and torch.equal(m.W, w1)
    m.switch_task("t1")
    # Omega = W / ((p - p_old)^2 + xi), by hand: 0.2 / (0.25 + 0.1), 0.1 / 0.35, 0 / 0.1, -0.3 / 1.1, ...
    omega1 = torch.tensor([0.2 / 0.35, 0.1 / 0.35, 0.0, -0.3 / 1.1, 0.05 / 0.14, 0.4 / 0.11, 0.0, 0.1 / 0.1])
    assert torch.allclose(m.F, omega1, rtol=1e-6)
    assert torch.equal(m.p_old, p1) and torch.count_nonzero(m.W) == 0 and m.task_name == "t1"
    assert torch.equal(m.Q, m.F) and torch.allclose(m.R, m.F * p1)
    p2 = p1 + torch.tensor([0.0, 1.0, 2.0, 0.0, -1.0, 0.0, 0.0, 0.5])
    w2 = torch.tensor([1.0, 0.2, 0.5, 0.0, 0.3, 0.0, -0.1, 0.0])
    a.master.copy_(p2)
    m.W.copy_(w2)
    m.switch_task("t2")
    omega2 = omega1 + torch.tensor([1.0 / 0.1, 0.2 / 1.1, 0.5 / 4.1, 0.0, 0.3 / 1.1, 0.0, -0.1 / 0.1, 0.0])
    assert torch.allclose(m.F, omega2, rtol=1e-6)                           # no clamping: negative entries stay
    assert torch.equal(m.p_old, p2) and torch.count_nonzero(m.W) == 0 and id(m.W) == W_id
    assert torch.allclose(m.penalty(), torch.tensor(0.0))
    a.master.add_(0.5)
    assert torch.allclose(m.penalty(), 0.5 * (omega2 * 0.25).sum())


@pytest.mark.parametrize("opts", [{"lambda_penalty": -1.0}, {"lambda_penalty": float("nan")},
                                  {"lambda_penalty": float("inf")}, {"si_xi": 0.0}, {"si_xi": -1e-3},
                                  {"si_xi": float("nan")}, {"lambda_penalty": "strong"}])
def test_bad_si_options_are_refused(opts):
    from flpr_b200.methods import si
    with pytest.raises(ValueError):
        si.Model(nn.Linear(3, 2), **opts)


def test_bad_si_option_is_refused_when_the_model_is_built():
    from flpr_b200.runtime.builder import parser_model
    cfg = dict(tiny_common("/nonexistent")["defaults"]["model_opts"], si_xi=0.0)
    with pytest.raises(ValueError):
        parser_model("si", cfg, "cpu")


def test_si_defaults():
    from flpr_b200.methods import si
    m = si.Model(nn.Linear(3, 2))
    assert m.lam == 0.1 and m.xi == 1e-3


def test_omega_is_refused_with_fedstil_terms():
    from flpr_b200.runtime.arena import ArenaOptimizer, ParamArena
    lin = nn.Linear(3, 2)
    arena = ParamArena(list(lin.named_parameters()), "cpu")
    opt = ArenaOptimizer("adam", arena)
    opt.omega = arena.new_buffer()
    opt.G = arena.master.clone()
    with pytest.raises(ValueError):
        opt.step()
    opt.G, opt.anchor = None, arena.master.clone()
    with pytest.raises(ValueError):
        opt.step()


# ------------------------------------------------------------------------------------------------ 4. penalty gradient
@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_penalty_gradient_on_the_second_task_matches_autograd(kind):
    """After a consolidation, one fused step (penalty folded into the kernel) equals an autograd step of
    ``torch.optim`` on ``loss + c * sum Omega (p - p_old)^2``; the path integral takes only the loss gradient."""
    from flpr_b200.runtime.arena import ArenaOptimizer
    c, lr = 0.7, 1e-2
    m = _tiny_si(lam=c)
    a = m.arena
    opt = ArenaOptimizer(kind, a, lr=lr)
    m.switch_task("t0")
    gen = torch.Generator().manual_seed(5)
    a.master.add_(torch.randn(a.numel, generator=gen) * 0.3)
    m.W.copy_(torch.rand(a.numel, generator=gen))
    m.switch_task("t1")
    assert torch.count_nonzero(m.F) == a.numel
    a.master.add_(torch.randn(a.numel, generator=gen) * 0.3)               # away from p_old: the penalty is active
    m.install(opt)
    assert opt.omega is m.W and opt.Q is m.Q and opt.R is m.R and opt.lam2 == c
    x, y = torch.randn(5, 2, generator=gen), torch.randn(5, 2, generator=gen)

    # reference: a leaf copy of the arena and torch.optim
    theta = a.master.clone().requires_grad_(True)
    omega, p_old = m.F.clone(), m.p_old.clone()
    ref_opt = (torch.optim.SGD if kind == "sgd" else torch.optim.Adam)([theta], lr=lr)
    w, b = theta[:4].view(2, 2), theta[4:6]
    loss = ((x @ w.t() + b - y) ** 2).mean()
    g_loss = torch.autograd.grad(loss, theta, retain_graph=True)[0]
    (loss + c * (omega * (theta - p_old) ** 2).sum()).backward()
    before = theta.detach().clone()
    ref_opt.step()

    opt.zero_grad()
    ((m.net(x) - y) ** 2).mean().backward()
    assert torch.allclose(a.grad, g_loss, rtol=1e-6, atol=1e-7)
    opt.step()
    assert torch.allclose(a.master, theta.detach(), rtol=1e-5, atol=1e-7)
    assert torch.allclose(m.W, -g_loss * (a.master - before), rtol=1e-4, atol=1e-9)


# -------------------------------------------------------------------------------------------- 5. end to end and resume
def _si_cfg(common, **over):
    mo = dict(common["defaults"]["model_opts"], lambda_penalty=1.0, si_xi=1e-3)
    return tiny_experiment(common, "si", n_tasks=3, model_opts=mo, **over)


def _si_run(tmp, emu=None):
    from flpr_b200.ops import native
    from flpr_b200.runtime.experiment import ExperimentStage
    common = tiny_common(str(tmp))
    common["defaults"]["exp_opts"].update(comm_rounds=3, val_interval=3)
    common["defaults"]["task_opts"]["sustain_rounds"] = 1
    cfg = _si_cfg(common)
    native.use_emulated_libraries(emu)
    try:
        before = native.launches()
        with ExperimentStage(common, [cfg], source_factory=tiny_factory()) as stage:
            log = stage.run_experiment(cfg)
        launches = native.launches() - before
    finally:
        native.use_emulated_libraries(None)
    return common, cfg, log, launches


def test_si_experiment_logs_and_checkpoint(tmp_path):
    common, cfg, log, _ = _si_run(tmp_path)
    data = log.records["data"]
    assert set(data) == {"client-0", "client-1"}
    for client, rounds in data.items():
        assert {"1", "2", "3"} <= set(rounds)
        for rnd in ("1", "2", "3"):
            task = f"task-{client[-1]}-{int(rnd) - 1}"
            assert {"tr_acc", "tr_loss"} <= set(rounds[rnd][task])
        assert {"val_rank_1", "val_map"} <= set(rounds["3"]["task-%s-0" % client[-1]])
    root = os.path.join(common["checkpoints_dir"], cfg["exp_name"])
    ck = torch.load(os.path.join(root, "client-0", "si_model.ckpt"), weights_only=False)
    assert set(ck) == {"net_params", "params_old", "precision_matrices", "path_integral"}
    assert set(ck["precision_matrices"]) == set(ck["params_old"]) == set(ck["path_integral"])
    assert "classifier.weight" in ck["precision_matrices"]
    omega = torch.cat([t.flatten() for t in ck["precision_matrices"].values()])
    W = torch.cat([t.flatten() for t in ck["path_integral"].values()])
    assert torch.count_nonzero(omega) > 0 and torch.count_nonzero(W) > 0   # two switches consolidated, task 3 live


def test_si_checkpoint_restores_all_four_parts():
    from flpr_b200.methods import si
    src = _tiny_si()
    for t in (src.F, src.p_old, src.W):
        t.copy_(torch.randn(src.arena.numel))
        t[6:] = 0                                       # arena padding: not part of the checkpoint
    src.arena.master.add_(1.0)
    state = src.model_state()
    dst = _tiny_si()
    W_id = id(dst.W)
    dst.update_model(state)
    assert isinstance(dst, si.Model) and id(dst.W) == W_id
    for name in ("F", "p_old", "W"):
        assert torch.equal(getattr(dst, name), getattr(src, name)), name
    assert torch.equal(dst.arena.master[:6], src.arena.master[:6])
    assert torch.equal(dst.R, dst.F * dst.p_old)


def test_si_experiment_on_the_emulated_kernels(tmp_path, emu_paths):
    def metrics(log):
        return {(c, r, t, k): float(v[k]) for c, per in log.records["data"].items() for r, ts in per.items()
                for t, v in ts.items() for k in ("tr_loss", "val_map", "val_rank_1") if k in v}
    *_, ref_log, n0 = _si_run(tmp_path / "ref")
    *_, got_log, n1 = _si_run(tmp_path / "emu", emu_paths)
    ref, got = metrics(ref_log), metrics(got_log)
    assert n0 == 0 and n1 >= 20, (n0, n1)
    assert ref.keys() == got.keys() and len(ref) >= 6
    for key in ref:
        assert abs(ref[key] - got[key]) <= 5e-3 * abs(ref[key]) + 1e-6, (key, ref[key], got[key])


def _resume_run(tmp, rounds, resume=False, interval=0):
    from flpr_b200.runtime import resume as R
    from flpr_b200.runtime.experiment import ExperimentStage
    from flpr_b200.runtime.explog import ExperimentLog
    from flpr_b200.utils.misc import DeviceTimer, same_seeds
    common = tiny_common(tmp)
    common["defaults"]["exp_opts"].update(comm_rounds=rounds, val_interval=100)
    common["defaults"]["task_opts"]["sustain_rounds"] = 1
    cfg = _si_cfg(common)
    cfg["engine_opts"].update(resume=resume, resume_interval=interval, val_at_round0=False)
    with ExperimentStage(common, [cfg], source_factory=tiny_factory()) as stage:
        same_seeds(cfg["random_seed"])
        store, comm, server, clients, names = stage.build(cfg)
        log = ExperimentLog(os.path.join(tmp, "log.json"), enabled=False)
        timer = DeviceTimer(stage.device)
        first = 1
        if resume and R.available(store, 0):
            first = R.load(stage, store, server, clients, comm) + 1
        for r in range(first, rounds + 1):
            stage._process_one_round(r, server, clients, names, cfg, log, timer, comm)
            if interval and r % interval == 0:
                R.save(stage, store, r, server, clients, comm)
        store.flush()
        out = {"clients": [c.model.arena.master.clone() for c in clients],
               "omega": [c.model.F.clone() for c in clients], "W": [c.model.W.clone() for c in clients],
               "task": [c.model.task_name for c in clients]}
        store.close()
        if comm is not None:
            comm.close()
    return out, first


def test_si_resume_across_a_task_switch(tmp_path):
    full, _ = _resume_run(str(tmp_path / "a"), 3)
    _, first = _resume_run(str(tmp_path / "b"), 1, interval=1)
    assert first == 1
    cont, first = _resume_run(str(tmp_path / "b"), 3, resume=True, interval=1)
    assert first == 2                                   # rounds 2 and 3 each start a new task after the restart
    assert cont["task"] == full["task"] == ["task-0-2", "task-1-2"]
    for key in ("clients", "omega", "W"):
        for a, b in zip(cont[key], full[key]):
            assert torch.allclose(a, b, atol=1e-5), key
    assert all(torch.count_nonzero(o) > 0 for o in full["omega"])

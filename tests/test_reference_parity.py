"""Golden parity against the UNMODIFIED reference: ranking metrics, distances, losses, FedAvg aggregation (incl. stale
clients) and the FedSTIL spatial-temporal mix. The reference's answers are stored under ``tests/golden/reference_parity``
(one file per test and oracle case, recorded by running ``tests/ref_oracle.py`` against the reference installed in
``oracle/_ref`` with ``FLPR_RECORD_GOLDEN=1``); every run compares this engine with them."""
import hashlib
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_parity")


def _golden_path(case):
    test = os.environ["PYTEST_CURRENT_TEST"].split(" ")[0].split("::", 1)[1]
    return os.path.join(GOLDEN, f"{hashlib.sha1(test.encode()).hexdigest()[:12]}_{case}.pt")


def oracle(case, payload, tmp_path):
    golden = _golden_path(case)
    if os.environ.get("FLPR_RECORD_GOLDEN") != "1":
        assert os.path.exists(golden), f"no stored reference answer {golden} (record it with FLPR_RECORD_GOLDEN=1)"
        return torch.load(golden, weights_only=False)
    inp, outp = str(tmp_path / f"{case}_in.pt"), str(tmp_path / f"{case}_out.pt")
    torch.save(payload, inp)
    env = dict(os.environ, TORCH_FORCE_NO_WEIGHTS_ONLY_LOAD="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "ref_oracle.py"), case, inp, outp],
                       capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    out = torch.load(outp, weights_only=False)
    os.makedirs(GOLDEN, exist_ok=True)
    torch.save(out, golden)
    return out


def test_ranking_metrics_match_reference(tmp_path):
    from flpr_b200.evaluation import evaluate
    torch.manual_seed(0)
    qf = torch.nn.functional.normalize(torch.randn(40, 64), dim=1)
    gf = torch.nn.functional.normalize(torch.randn(150, 64), dim=1)
    ql, gl = torch.randint(0, 12, (40,)), torch.randint(0, 12, (150,))
    ref = oracle("evaluate", {"qf": qf, "ql": ql, "gf": gf, "gl": gl}, tmp_path)
    cmc, mAP = evaluate(qf, ql, gf, gl)
    assert abs(float(mAP) - ref["mAP"]) < 1e-5
    assert torch.allclose(torch.as_tensor(cmc).float()[:len(ref["cmc"])], ref["cmc"], atol=1e-5)
    # CMC is unaffected by the modern-stack argwhere quirk of the reference; its "mAP" degenerates to first-hit precision
    assert torch.allclose(ref["raw_cmc"], ref["cmc"], atol=1e-6) and ref["raw_mAP"] != pytest.approx(ref["mAP"])


def test_camera_junk_rule():
    """Optional camera labels: same identity under the query's camera and label -1 are junk (evaluate.py:12-33,60-67).
    The reference's own camera branch cannot run - ``np.setdiff1d`` hands ``evaluate_with_index`` a flat array and
    ``len(right_result_index[0])`` raises ``TypeError`` - so the rule is checked against a literal per-query
    re-statement of it (sort, drop junk, locate hits, trapezoid AP)."""
    import numpy as np
    from flpr_b200.evaluation import evaluate
    torch.manual_seed(3)
    qf = torch.nn.functional.normalize(torch.randn(30, 48), dim=1)
    gf = torch.nn.functional.normalize(torch.randn(120, 48), dim=1)
    ql, gl = torch.randint(0, 8, (30,)), torch.randint(0, 8, (120,))
    gl[::17] = -1                                                     # mis-detections
    qc, gc = torch.randint(0, 3, (30,)), torch.randint(0, 3, (120,))
    cmc, mAP = evaluate(qf, ql, gf, gl, qc, gc)
    sim = (qf @ gf.t()).numpy()
    total_cmc, total_ap = np.zeros(120), 0.0
    for i in range(30):
        order = np.argsort(sim[i])[::-1]
        same_id, same_cam = gl.numpy() == int(ql[i]), gc.numpy() == int(qc[i])
        junk = np.flatnonzero((same_id & same_cam) | (gl.numpy() == -1))
        right = np.flatnonzero(same_id & ~same_cam)
        if right.size == 0:
            continue
        order = order[np.isin(order, junk, invert=True)]
        loc = np.flatnonzero(np.isin(order, right))
        total_cmc[loc[0]:] += 1
        total_ap += sum(((j / l if l else 1.0) + (j + 1) / (l + 1)) / 2 for j, l in enumerate(loc)) / right.size
    assert np.allclose(cmc, total_cmc / 30, atol=1e-9) and abs(mAP - total_ap / 30) < 1e-9
    plain_cmc, plain_map = evaluate(qf, ql, gf, gl)
    assert abs(plain_map - mAP) > 1e-3                                 # the rule does change the numbers here


def test_accuracy_and_forgetting_tables_match_reference(tmp_path):
    """``analyse/accuracy.py::accuracy_on_round`` / ``analyse/forgetting.py::forgetting_on_round`` print per-client and
    total percentages; the same log dict must give the same lines."""
    import contextlib
    import io
    import random
    from flpr_b200.analyse.accuracy import accuracy_on_round
    from flpr_b200.analyse.forgetting import forgetting_on_round
    rng = random.Random(4)
    logs = {}
    for c in range(3):
        logs[f"client-{c}"] = {str(r): {f"task-{c}-{t}": {"val_map": rng.random(), "val_rank_1": rng.random(),
                                                          **({"tr_acc": rng.random()} if t == min(r // 2, 2) else {})}
                                           for t in range(3) if t <= r // 2 + 1} for r in range(0, 7)}
    ref = oracle("analyse", {"logs": logs, "rounds": [2, 4, 6], "metric": "val_map"}, tmp_path)
    for rnd in (2, 4, 6):
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            accuracy_on_round(logs, rnd, "val_map", "metric")
            forgetting_on_round(logs, rnd, "val_map", "metric")
        assert buf.getvalue() == ref[rnd], (buf.getvalue(), ref[rnd])


def test_task_schedule_matches_reference(tmp_path):
    """``ReIDTaskPipeline.next_task`` (datasets_pipeline.py:81-93): ``sustain_rounds`` rounds per task, then the last
    task forever; index, remaining-round counters and ``reach_final_task`` after every call."""
    from flpr_b200.data.pipeline import ReIDTaskPipeline
    tasks = ["task-0-0", "task-0-1", "task-0-2"]
    ref = oracle("schedule", {"tasks": tasks, "sustain": [1, 2, 3], "calls": 14}, tmp_path)
    for sustain in (1, 2, 3):
        pipe = ReIDTaskPipeline(list(tasks), {"sustain_rounds": sustain}, "unused")
        pipe.get_task = lambda idx=-1: pipe.task_list[idx]
        seq = [(pipe.next_task(), pipe.current_task_idx, list(pipe.task_round_rest), pipe.reach_final_task())
               for _ in range(14)]
        assert seq == [tuple(x) for x in ref[sustain]], sustain


def test_experiment_log_record_semantics_match_reference(tmp_path):
    """``ExperimentLog.record`` (experiment.py:16-55): dotted keys create nested dicts; an existing list is appended to,
    a set added to, a dict updated, anything else replaced - and the JSON file mirrors the records."""
    import json
    from flpr_b200.runtime.explog import ExperimentLog
    ops = [("config", {"exp_name": "x", "seed": 1}), ("data.client-0.1.task-0-0", {"tr_acc": 0.5, "tr_loss": 2.0}),
           ("data.client-0.1.task-0-0", {"val_map": 0.25}), ("data.client-0.2.task-0-0", {"tr_acc": 0.75}),
           ("data.client-1.1.task-1-0", {"val_rank_1": 0.1}), ("notes", [1]), ("notes", 2), ("scalar", 3), ("scalar", 4),
           ("config", {"seed": 2})]
    ref = oracle("explog", {"path": str(tmp_path / "ref.json"), "ops": ops}, tmp_path)
    log = ExperimentLog(str(tmp_path / "mine.json"))
    for key, value in ops:
        log.record(key, value)
    log.flush() if hasattr(log, "flush") else None
    assert log.records == ref["records"]
    assert json.load(open(tmp_path / "mine.json")) == ref["file"]


def test_console_line_formats_match_reference(tmp_path):
    """``tools/logger.py:23-39``: the formatted train line and validation block, character for character."""
    import logging
    from flpr_b200.utils.logger import Logger
    cmc = [0.1 * i for i in range(1, 11)]
    ref = oracle("logger", {"cmc": cmc}, tmp_path)
    msgs = []

    class _H(logging.Handler):
        def emit(self, record):
            msgs.append(record.getMessage())

    lg = Logger("client-0-format-test")
    handler = _H()
    lg.logger.addHandler(handler)
    lg.logger.setLevel(logging.INFO)
    try:
        lg.info_train("task-0-1", "cuda:0", 12345, 0.98765, 1.23456, 3, 5)
        lg.info_train("task-0-1", "cpu", 7, 0.5, 0.25)
        lg.info_validation("task-0-1", 1234, 56789, cmc, 0.4321)
    finally:
        lg.logger.removeHandler(handler)
    assert msgs == ref


def test_distances_match_reference(tmp_path):
    from flpr_b200 import criterions as C
    torch.manual_seed(1)
    a, b = torch.randn(6, 32), torch.randn(9, 32)
    ref = oracle("distance", {"a": a, "b": b}, tmp_path)
    assert torch.allclose(C.euclidean_dist(a, b), ref["eu"], atol=1e-4)
    assert torch.allclose(C.cosine_dist(a, b), ref["cos"], atol=1e-5)
    assert torch.allclose(C.kl_distance(a[:1], b[:1]), ref["kl"], atol=1e-5)


def test_losses_match_reference(tmp_path):
    from flpr_b200.criterions import criterions
    torch.manual_seed(2)
    score, feat = torch.randn(16, 50), torch.randn(16, 24)
    target = torch.arange(16) % 4
    teacher = torch.randn(16, 50)
    ref = oracle("losses", {"score": score, "feat": feat, "target": target, "teacher": teacher, "T": 4.0}, tmp_path)
    kd = criterions["kd_loss"](temperature=4.0)
    assert torch.allclose(kd(score, teacher), ref["kd"], atol=1e-5)
    assert torch.allclose(kd(score=score, teacher_score=teacher), ref["kd"], atol=1e-5)
    s = score.clone().requires_grad_(True)
    ce = criterions["cross_entropy"](num_classes=50, epsilon=0.1)
    loss = ce(score=s, feature=None, target=target)
    loss.backward()
    assert torch.allclose(loss.detach(), ref["ce"], atol=1e-5) and torch.allclose(s.grad, ref["ce_grad"], atol=1e-6)
    for name, kw in (("tri_hard", dict(margin=0.3, hard_mining=True)), ("tri_soft", dict(margin=0, hard_mining=True)),
                     ("tri_w", dict(margin=0.3, hard_mining=False, norm_feat=True))):
        t = criterions["triplet_loss"](**kw)
        assert torch.allclose(t(score=None, feature=feat, target=target), ref[name], atol=1e-5), name


def test_fedavg_aggregation_matches_reference_incl_stale_clients(tmp_path):
    """Same uploads -> same weighted mean; a client that did not upload this round keeps contributing its old state."""
    from flpr_b200.parallel.comm import FedComm
    torch.manual_seed(3)
    shapes = {"w1": (7, 5), "b1": (7,), "w2": (3, 7)}
    n = sum(torch.Size(s).numel() for s in shapes.values())
    n_pad = (n + 3) // 4 * 4
    clients, flat = {}, {}
    for cid, (name, k) in enumerate((("c0", 48), ("c1", 16), ("c2", 80))):
        params = {pn: torch.randn(*s) for pn, s in shapes.items()}
        clients[name] = {"train_cnt": k, "incremental_model_params": params}
        flat[cid] = torch.cat([p.flatten() for p in params.values()] + [torch.zeros(n_pad - n)])
    ref = oracle("fedavg_calculate", {"clients": clients}, tmp_path)
    comm = FedComm("cpu", 3, arena_bytes=1 << 20)
    comm.alloc_client_buffer("up", n_pad)
    comm.alloc_client_buffer("cnt", 4)
    comm.alloc_rank_buffer("glob", n_pad)
    for cid, (name, st) in enumerate(clients.items()):
        comm.client_view("up", cid).copy_(flat[cid])
        comm.client_view("cnt", cid).fill_(float(st["train_cnt"]))
    comm.reduce_bcast("up", "glob", [0, 1, 2], cnt="cnt")
    got = comm.rank_view("glob")[:n]
    want = torch.cat([ref[pn].flatten() for pn in shapes])
    assert torch.allclose(got, want, atol=1e-5)
    comm.close()


def test_fedstil_mix_matches_reference(tmp_path):
    """Decayed-KL relevance -> own = mean -> normalise -> softmax -> per-client weighted parameter mix."""
    from flpr_b200.methods.fedstil import Server
    torch.manual_seed(4)
    names = ["c0", "c1", "c2", "c3"]
    theta = {n: {"l.global_weight": torch.randn(6, 4), "m.global_weight": torch.randn(5)} for n in names}
    mem = {n: [torch.randn(40) for _ in range(5)] for n in names}
    clients = {n: {"task_token": mem[n][-1], "incremental_sw": theta[n], "train_cnt": 10} for n in names}
    ref = oracle("fedstil_dispatch", {"clients": clients, "token_memory": mem, "step": 2, "decay": 0.8,
                                      "receivers": names}, tmp_path)
    srv = Server.__new__(Server)
    srv.distance_calculate_step, srv.distance_calculate_decay = 2, 0.8
    srv.token_memory = mem
    order, W = srv.relevance_rows(names)
    for r, name in enumerate(names):
        for key in ("l.global_weight", "m.global_weight"):
            mixed = sum(W[r, order.index(c)] * theta[c][key] for c in names)
            assert torch.allclose(mixed, ref[name][key], atol=1e-5), (name, key)


def test_swin_transformer_matches_reference(tmp_path):
    """Same state dict (key-compatible) -> same features / logits as the reference Swin implementation, on both the
    fused-attention code path (tensor-op form on CPU) and the SDPA path (shifted windows, masks, patch merging)."""
    from flpr_b200.models.swin import SwinTransformer, WindowAttention
    torch.manual_seed(5)
    net = SwinTransformer(img_size=56, embed_dim=24, depths=(2, 2), num_heads=(2, 4), window_size=7, num_classes=5,
                          drop_path_rate=0.0).eval()
    cfg = {"img": 56, "dim": 24, "depths": (2, 2), "heads": (2, 4), "ws": 7, "classes": 5,
           "x": torch.randn(2, 3, 56, 56), "state": net.state_dict()}
    ref = oracle("swin_forward", cfg, tmp_path)
    # the reference module takes this engine's state dict: every parameter / buffer key exists on both sides
    assert not [k for k in ref["missing"] if "relative_position_index" not in k and "attn_mask" not in k], ref["missing"]
    assert not [k for k in ref["unexpected"] if not k.endswith(("relative_position_index", "attn_mask"))], ref["unexpected"]
    for fused in (True, False):
        for m in net.modules():
            if isinstance(m, WindowAttention):
                m.fused = fused
        with torch.no_grad():
            assert torch.allclose(net.forward_features(cfg["x"]), ref["feat"], atol=2e-5), fused
            assert torch.allclose(net(cfg["x"]), ref["logits"], atol=2e-5), fused


def test_fedcurv_three_moment_penalty_matches_reference(tmp_path):
    """The reference ships (1 + 2K) parameter-sized tensors to every client and loops over them in ``penalty()``
    (fedcurv.py:79-86, 621-646). Here the server pre-reduces three moments (sum F_j, sum F_j p_j, sum F_j p_j^2) and
    the optimizer kernel uses ``2 lam (Q p - R)``: same gradient, same value (up to the constant moment)."""
    import torch.nn as nn
    from flpr_b200.methods.fedcurv import Model
    from flpr_b200.ops.fused import fused_optimizer_step
    from flpr_b200.parallel.comm import FedComm
    torch.manual_seed(6)
    net = nn.Sequential(nn.Linear(6, 5), nn.Linear(5, 3))
    model = Model(net, lambda_penalty=7.0).materialize("cpu", "fp32", None)
    a = model.arena
    names = list(a.segments.keys())
    n = a.numel

    def rnd_dict(pos=False):
        return {k: (torch.rand_like(a.view(a.master, k)) if pos else torch.randn_like(a.view(a.master, k)))
                for k in names}

    F_own, p_old = rnd_dict(True), rnd_dict()
    others = [(rnd_dict(True), rnd_dict()) for _ in range(3)]
    params = {k: a.view(a.master, k).detach().clone() for k in names}
    ref = oracle("fedcurv_penalty", {"lam": 7.0, "params": params, "F": F_own, "p_old": p_old, "others": others},
                 tmp_path)
    # ours: own Fisher / old params into the model, the others' (F_j, p_j) through the moment collective
    a.from_dict(F_own, model.F)
    a.from_dict(p_old, model.p_old)
    comm = FedComm("cpu", 3, arena_bytes=1 << 20)
    for nm in ("fisher", "param"):
        comm.alloc_client_buffer(nm, n)
    for nm in ("mf", "mfp", "mfpp"):
        comm.alloc_rank_buffer(nm, n)
    for cid, (Fj, pj) in enumerate(others):
        a.from_dict(Fj, comm.client_view("fisher", cid))
        a.from_dict(pj, comm.client_view("param", cid))
    comm.curv_moments("fisher", "param", [0, 1, 2], "mf", "mfp", "mfpp")
    model.set_others(comm.rank_view("mf"), comm.rank_view("mfp"), comm.rank_view("mfpp"))
    const = float((model.F * model.p_old ** 2).sum() * 0 + comm.rank_view("mfpp").sum())     # sum_j F_j p_j^2
    assert abs(float(model.penalty()) + 7.0 * const - float(ref["value"])) < 1e-3 * abs(float(ref["value"]))
    # gradient of the penalty as the fused optimizer sees it: plain SGD step with lr = 1, zero data gradient
    p0 = a.master.clone()
    g = torch.zeros_like(p0)
    fused_optimizer_step("sgd", a.master, g, None, None, lr=1.0, step=1, Q=model.Q, R=model.R, lam2=model.lam)
    grad_flat = p0 - a.master
    for k in names:
        assert torch.allclose(a.view(grad_flat, k), ref["grads"][k], rtol=1e-4, atol=1e-4), k
    comm.close()


@pytest.mark.parametrize("opt,wd,steps", [("sgd", 0.0, 3), ("adam", 0.0, 2), ("adam", 1e-2, 1)])
def test_fedstil_theta_training_equals_reference_adaptive_layer(tmp_path, opt, wd, steps):
    """Training ``theta`` directly with the fused optimizer (weight decay on ``theta - a G``, L1 ``sign(theta - G)``)
    reproduces the reference's ``AdaptiveLayer`` (frozen ``atten (.) G`` + trained ``A``, L1 towards ``A0``).
    With weight decay the reference also moves its accidentally trainable ``initial_*`` copies (a documented deviation),
    which only matters from the second step on."""
    from flpr_b200.ops.fused import fused_optimizer_step
    torch.manual_seed(8)
    G = torch.randn(5, 7)
    xs = [torch.randn(4, 7) for _ in range(steps)]
    ts = [torch.randn(4, 5) for _ in range(steps)]
    a, lr, lam1 = 0.8, 0.05, 1e-2
    ref = oracle("fedstil_layer_steps", {"G": G, "atten": a, "lr": lr, "wd": wd, "opt": opt, "lam1": lam1,
                                         "xs": xs, "ts": ts}, tmp_path)
    theta = G.clone().flatten()
    Gf = G.clone().flatten()
    m, v = torch.zeros_like(theta), torch.zeros_like(theta)
    for i, (x, t) in enumerate(zip(xs, ts)):
        th = theta.view(5, 7).clone().requires_grad_(True)
        ((torch.nn.functional.linear(x, th) - t) ** 2).mean().backward()
        fused_optimizer_step(opt, theta, th.grad.flatten().clone(), m, v, lr=lr, step=i + 1, weight_decay=wd, G=Gf,
                             lam1=lam1, atten=a)
        assert torch.allclose(theta.view(5, 7), ref["thetas"][i], atol=2e-6), (opt, i)


# Adam with the shipped weight decay (1e-5: the anchor's gradient is of the order of Adam's eps, so anchor and weight
# separate by ~lr/2 at once). With a large decay both move by lr * (1 - eps/|g|) and sign(aw - aw0) is decided by a
# 1e-7-sized difference - the reference's own trajectory is then a matter of fp32 rounding order, nothing to match.
@pytest.mark.parametrize("opt,wd,steps", [("sgd", 1e-2, 6), ("adam", 1e-5, 6), ("adam", 0.0, 6)])
def test_fedstil_trained_anchor_matches_reference_adaptive_layer(tmp_path, opt, wd, steps):
    """``engine_opts.train_l1_anchor``: with the L1 anchor trained like the reference's optimizer trains its
    ``initial_adaptive_weight`` (gradient ``-lam1 sign(aw - aw0) + wd aw0``), the theta trajectory follows the
    reference's ``AdaptiveLayer`` over many steps, weight decay included."""
    import torch.nn as nn
    from flpr_b200.runtime.arena import ArenaOptimizer, ParamArena
    torch.manual_seed(8)
    G = torch.randn(5, 7)
    xs = [torch.randn(4, 7) for _ in range(steps)]
    ts = [torch.randn(4, 5) for _ in range(steps)]
    a, lr, lam1 = 0.8, 0.05, 1e-2
    ref = oracle("fedstil_layer_steps", {"G": G, "atten": a, "lr": lr, "wd": wd, "opt": opt, "lam1": lam1,
                                         "xs": xs, "ts": ts}, tmp_path)
    lin = nn.Linear(7, 5, bias=False)
    with torch.no_grad():
        lin.weight.copy_(G)
    arena = ParamArena([("weight", lin.weight)], "cpu")
    optim = ArenaOptimizer(opt, arena, lr=lr, weight_decay=wd)
    optim.G, optim.lam1, optim.atten = G.clone().flatten(), lam1, a
    optim.anchor = optim.G.clone()
    optim.stats = torch.zeros(2)
    for i, (x, t) in enumerate(zip(xs, ts)):
        optim.zero_grad()
        ((lin(x) - t) ** 2).mean().backward()
        optim.step()
        assert torch.allclose(lin.weight.detach(), ref["thetas"][i], atol=5e-6), (opt, i)
    assert float(optim.stats[1]) > 0                      # sum |aw - aw0| is still reported


@pytest.mark.parametrize("method", ["ewc", "mas", "fedcurv"])
def test_importance_accumulation_matches_reference(tmp_path, method):
    """Fisher (g^2) / MAS (|g|) importance over the remembered loaders with the reference's ``len(batch) / #batches``
    weighting; EWC skips the most recent task (ewc.py:62-65), MAS and FedCurv do not."""
    import torch.nn as nn
    import torch.nn.functional as F
    from flpr_b200.methods import methods
    torch.manual_seed(9)
    net = nn.Sequential(nn.Linear(6, 5), nn.ReLU(), nn.Linear(5, 4))
    state = {k: v.clone() for k, v in net.state_dict().items()}
    loaders = {f"task-{t}": [(torch.randn(bs, 6), torch.randint(0, 4, (bs,))) for bs in (5, 3, 4)] for t in range(3)}
    ref = oracle("importance", {"method": method, "state": state, "loaders": loaders}, tmp_path)

    class Op:
        def _invoke_train(self, model, data, target, **kw):
            return {"loss": F.cross_entropy(model(data), target)}

    model = methods[method].Model(net, operator=Op()).materialize("cpu", "fp32", None)

    class Loader(list):
        pass
    for name, batches in loaders.items():
        model.recall_dataloaders[name] = Loader([(x, y, y) for x, y in batches])
    model._calculate_importance()
    got = model.arena.to_dict(model.F)
    for k, v in ref.items():
        assert torch.allclose(got[k], v, rtol=1e-4, atol=1e-6), (method, k)

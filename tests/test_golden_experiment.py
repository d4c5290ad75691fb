"""Whole-experiment golden parity (SURVEY §7.4): the UNMODIFIED reference (``oracle/_ref``, subprocess) and this engine
run the same tiny fp32 CPU experiment – same initial weights, same synthetic splits, every split smaller than one batch
so the reference's shuffling cannot change the arithmetic – and every payload / model checkpoint the reference wrote is
compared tensor by tensor with the file this engine wrote under the same name."""
import copy
import os
import subprocess
import sys

import pytest
import torch

from flpr_b200.data.datasets import ArrayReIDDataset
from flpr_b200.runtime.config import merge_experiment
from flpr_b200.runtime.experiment import ExperimentStage

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
pytestmark = pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "methods")),
                                reason="the reference oracle is not built in oracle/_ref")

H, W, CLIENTS, TASKS, ROUNDS = 32, 16, 2, 2, 2
# The default run keeps the suite around ten minutes on a CPU box; FLPR_GOLDEN_FULL=1 adds the remaining variants.
OVERRIDES: dict = {}        # per-test overrides of the shared config (epochs, lr); see test_early_stopping_...
full = pytest.mark.skipif(os.environ.get("FLPR_GOLDEN_FULL") != "1", reason="set FLPR_GOLDEN_FULL=1 for the full matrix")


def _common(tmp: str, rounds: int = ROUNDS, online: int = CLIENTS, adam: bool = False):
    epochs, sgd_lr = OVERRIDES.get("epochs", 2), OVERRIDES.get("lr", 0.05)
    criteria = [{"name": "cross_entropy", "num_classes": 8000, "epsilon": 0.1}] + list(OVERRIDES.get("extra_criteria", []))
    return {"datasets_dir": os.path.join(tmp, "data"), "checkpoints_dir": os.path.join(tmp, "ckpts"),
            "logs_dir": os.path.join(tmp, "logs"), "parallel": 1, "device": ["cpu"],
            "defaults": {
                "random_seed": 7,
                "exp_opts": {"comm_rounds": rounds, "val_interval": 1, "online_clients": online},
                "model_opts": {"name": "resnet18", "num_classes": 8000, "last_stride": 1, "neck": "bnneck",
                               "fine_tuning": ["base.layer4", "classifier"]},
                "criterion_opts": criteria[0] if len(criteria) == 1 else criteria,
                # SGD + momentum: an update is proportional to the gradient, so a rounding-level difference stays a
                # rounding-level difference. ``adam=True`` runs the reference's default optimizer instead.
                "optimizer_opts": ({"name": "adam", "lr": 1e-3, "weight_decay": 1e-5} if adam else
                                   {"name": "sgd", "lr": sgd_lr, "momentum": 0.9, "weight_decay": 1e-4}),
                "scheduler_opts": {"name": "step_lr", "step_size": OVERRIDES.get("step_size", 5)},
                "task_opts": {"sustain_rounds": 1, "train_epochs": epochs,
                              "augment_opts": {"level": "none", "img_size": [H, W],
                                               "norm_mean": [0.485, 0.456, 0.406], "norm_std": [0.229, 0.224, 0.225]},
                              "loader_opts": {"batch_size": 32, "num_workers": 0, "pin_memory": False,
                                              "persistent_workers": False, "multiprocessing_context": None}}}}


METHOD_OPTS = {
    "fedstil": dict(atten_default=0.9, lambda_l1=1e-4, lambda_k=8),
    "fedstil-atten": dict(atten_default=0.5, lambda_l1=1e-5, lambda_k=8),
    "fedweit": dict(lambda_l1=1e-3, lambda_l2=100.0, lambda_mask=0.0, kb_cnt=2),
    "fedprox": dict(lambda_l2=1e-2),
    "fedcurv": dict(lambda_penalty=10.0),
    "ewc": dict(lambda_penalty=50.0),
    "mas": dict(lambda_penalty=0.01),
    "icarl": dict(k=8, n_classes=50),
}


def _experiment(common, method):
    backbone, shared_ckpt = None, None
    if "@" in method:                                   # "fedstil@swin_transformer_tiny"
        method, backbone = method.split("@")
    if "+" in method:                                   # "baseline+sm_model": one shared checkpoint name (config "sm")
        method, shared_ckpt = method.split("+")
    exp = {"exp_name": f"golden-{method}", "exp_method": method, "server": {"server_name": "server"},
           "clients": [{"client_name": f"client-{i}", "tasks": [f"task-{i}-{t}" for t in range(TASKS)]}
                       for i in range(CLIENTS)]}
    if method in METHOD_OPTS:
        exp["model_opts"] = dict(common["defaults"]["model_opts"], **METHOD_OPTS[method])
    if method.startswith("fedstil"):
        exp["server"].update(distance_calculate_step=1, distance_calculate_decay=0.8)
        for c in exp["clients"]:
            c["model_ckpt_name"] = "fedstil_model"
    if shared_ckpt is not None:
        for c in exp["clients"]:
            c["model_ckpt_name"] = shared_ckpt
    if backbone is not None:
        exp["model_opts"] = dict(exp.get("model_opts") or common["defaults"]["model_opts"], name=backbone,
                                 fine_tuning=["base.layers.3", "classifier"] if "swin" in backbone
                                 else ["base.layer4", "classifier"])
        if "swin" in backbone:
            exp["model_opts"]["drop_path_rate"] = 0.0           # see tests/ref_golden.py
    return exp


def _splits():
    g = torch.Generator().manual_seed(99)
    out = {}
    for c in range(CLIENTS):
        for t in range(TASKS):
            off = 10 * (c * TASKS + t)
            for split, n in (("train", 12), ("query", 4), ("gallery", 12)):
                u8 = torch.randint(0, 256, (n, H, W, 3), dtype=torch.uint8, generator=g)
                pids = torch.arange(n) % 4 + off
                out[(f"task-{c}-{t}", split)] = (u8, pids)
    return out


def _run_reference(tmp_path, method, splits, rounds=ROUNDS, online=CLIENTS, adam=False, val0=False):
    tmp = str(tmp_path / "ref")
    os.makedirs(tmp)
    common = _common(tmp, rounds, online, adam)
    exp = dict(copy.deepcopy(common["defaults"]))
    exp.update(_experiment(common, method))
    inp, outp = os.path.join(tmp, "in.pt"), os.path.join(tmp, "out.pt")
    torch.save({"common": common, "exp": exp, "rounds": rounds, "splits": splits, "val0": val0}, inp)
    env = dict(os.environ, TORCH_FORCE_NO_WEIGHTS_ONLY_LOAD="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "ref_golden.py"), inp, outp], capture_output=True,
                       text=True, env=env, timeout=900, cwd=tmp)
    assert r.returncode == 0, r.stderr[-3000:]
    return torch.load(outp, weights_only=False)


def _run_ours(tmp_path, method, splits, init, rounds=ROUNDS, online=CLIENTS, adam=False, engine=None):
    tmp = str(tmp_path / "ours")
    os.makedirs(tmp)
    common = _common(tmp, rounds, online, adam)
    init_path = os.path.join(tmp, "init.pt")
    torch.save(init, init_path)
    exp = _experiment(common, method)
    method = method.split("@")[0].split("+")[0]
    exp["engine_opts"] = {"compute_dtype": "fp32", "init_state": init_path, "val_at_round0": False,
                          "client_threads": False, **(engine or {})}
    cfg = merge_experiment(common, exp)

    def factory(task, split):
        u8, pids = splits[(task, split)]
        return ArrayReIDDataset(u8, pids, pin=False)

    with ExperimentStage(common, [cfg], source_factory=factory) as stage:
        log = stage.run_experiment(cfg)
    root = os.path.join(common["checkpoints_dir"], cfg["exp_name"])
    files = {}
    for dirpath, _, names in os.walk(root):
        for n in names:
            if n.endswith(".ckpt"):
                p = os.path.join(dirpath, n)
                files[os.path.relpath(p, root)] = torch.load(p, map_location="cpu", weights_only=False)
    return files, log.records


# Parameters / buffers owned by NON-leaf modules. The reference's ``pre_trained_params`` enumerates leaf modules only
# (fedstil.py:482-486), so it neither checkpoints nor dispatches them; this engine writes them too (strict superset).
SWIN_EXTRA = ("relative_position_bias_table", "relative_position_index", "attn_mask")


def _compare(path, a, b, atol, rtol, bad, ignore=(), max_factor=10):
    """Recursive comparison of two checkpoint objects (``a`` = reference); mismatches are appended to ``bad``.
    ``ignore``: dict keys of the reference that this engine deliberately does not materialise."""
    import numpy as np
    if isinstance(a, dict):
        a = {k: v for k, v in a.items() if str(k) not in ignore}
        if isinstance(b, dict):                 # documented supersets (SWIN_EXTRA): keys only this engine writes
            b = {k: v for k, v in b.items() if str(k) in map(str, a) or not str(k).endswith(SWIN_EXTRA)}
        if not isinstance(b, dict) or set(map(str, a)) != set(map(str, b)):
            bad.append((path, "keys", sorted(map(str, a))[:6], sorted(map(str, b))[:6] if isinstance(b, dict) else type(b)))
            return
        bk = {str(k): v for k, v in b.items()}
        for k, v in a.items():
            _compare(f"{path}/{k}", v, bk[str(k)], atol, rtol, bad, ignore, max_factor)
    elif isinstance(a, (list, tuple)):
        if not isinstance(b, (list, tuple)) or len(a) != len(b):
            bad.append((path, "len", len(a), len(b) if hasattr(b, "__len__") else type(b)))
            return
        for i, (x, y) in enumerate(zip(a, b)):
            _compare(f"{path}[{i}]", x, y, atol, rtol, bad, ignore, max_factor)
    elif isinstance(a, (torch.Tensor, np.ndarray)):
        ta, tb = torch.as_tensor(a).float(), torch.as_tensor(b).float()
        if ta.shape != tb.shape:
            bad.append((path, "shape", tuple(ta.shape), tuple(tb.shape)))
        elif not torch.allclose(ta, tb, atol=atol, rtol=rtol):
            # Both sides run the same ATen kernels, but the reference shuffles its (single) batch differently, so
            # batch-statistic sums round differently; a pre-activation within ~1e-7 of zero then takes the other
            # ReLU branch (or an |aw - aw0| ~ 0 element the other L1 sub-gradient sign) and a handful of weights move
            # by up to lr * |grad|. Those isolated elements are tolerated; a systematic difference is not.
            d = (ta - tb).abs()
            outliers = float((d > atol + rtol * ta.abs()).float().mean())
            amax = float(ta.abs().max())
            diffuse = float(d.max()) <= 5 * (atol + rtol * amax)     # e.g. BN running statistics downstream of a flip
            sparse = float(d.max()) <= max_factor * atol + rtol * amax and outliers <= 0.05
            if not (diffuse or sparse):
                bad.append((path, "value", float(d.max()), float(ta.abs().max()), f"outliers {outliers:.4f}"))
    elif isinstance(a, (int, float)):
        if abs(float(a) - float(b)) > atol + rtol * abs(float(a)):
            bad.append((path, "scalar", a, b))
    elif a is None:
        if b is not None:
            bad.append((path, "none", a, type(b)))


def golden(tmp_path, method, atol=2e-5, rtol=1e-4, skip=(), ignore=(), rounds=ROUNDS, max_factor=10, online=None,
           adam=False, engine=None, clients=None, tasks=None, val0=False):
    import shutil
    global CLIENTS, TASKS
    saved, CLIENTS = CLIENTS, clients or CLIENTS            # _splits / _experiment read the module-level counts
    saved_t, TASKS = TASKS, tasks or TASKS
    try:
        return _golden(tmp_path, method, atol, rtol, skip, ignore, rounds, max_factor, online or CLIENTS, adam, engine,
                       val0)
    finally:
        CLIENTS, TASKS = saved, saved_t


def _golden(tmp_path, method, atol, rtol, skip, ignore, rounds, max_factor, online, adam, engine, val0=False):
    import shutil
    splits = _splits()
    ref = _run_reference(tmp_path, method, splits, rounds, online, adam, val0)
    shutil.rmtree(tmp_path / "ref", ignore_errors=True)           # hundreds of MB of checkpoints per run
    if val0:
        engine = dict(engine or {}, val_at_round0=True)
    files, log = _run_ours(tmp_path, method, splits, ref["init"], rounds, online, adam, engine)
    shutil.rmtree(tmp_path / "ours", ignore_errors=True)
    bad = []
    missing = [f for f in ref["files"] if f not in files]
    assert not missing, f"files the reference wrote and this engine did not: {missing}"
    for name, obj in sorted(ref["files"].items()):
        if any(s in name for s in skip):
            continue
        _compare(name, obj, files[name], atol, rtol, bad, ignore, max_factor)
    assert not bad, "\n".join(map(str, bad[:20]))
    # logged metrics (tr_acc / tr_loss / CMC / mAP) of every client, round and task
    for client, rounds in ref["log"].get("data", {}).items():
        for rnd, tasks in rounds.items():
            for task, metrics in tasks.items():
                mine = log["data"][client][str(rnd)][task]
                for k, v in metrics.items():
                    assert abs(float(mine[k]) - float(v)) < 1e-3, (client, rnd, task, k, v, mine[k])
    return ref, files


# FedCurv: the reference materialises every other client's (F_j, p_j) in its dispatch payload and model checkpoint; this
# engine exchanges three pre-reduced moment buffers instead (methods/fedcurv.py) - everything else is compared.
FEDCURV_NOT_MATERIALISED = ("other_precision_matrices", "other_clients_integrated_params",
                            "other_clients_incremental_params", "other_clients_precision_matrices")


@pytest.mark.parametrize("method", ["baseline", "ewc", "mas", "fedprox", "fedcurv", "fedweit", "fedstil-atten"])
def test_experiment_matches_reference(tmp_path, method):
    golden(tmp_path, method, ignore=FEDCURV_NOT_MATERIALISED if method == "fedcurv" else ())


@pytest.mark.parametrize("method", ["fedavg", "fedstil", pytest.param("fedweit", marks=full)])
def test_three_rounds_match_reference(tmp_path, method):
    """Third round = second round on the last task (stickiness) and the 5th / 6th epoch: crosses the StepLR boundary
    (and the reference's per-epoch lr reset in fedweit / fedstil), evaluates FedWeIT's older task from its own
    checkpoint, and for FedSTIL rehearses exemplars of two tasks (the class-index relabelling quirk)."""
    if method == "fedstil":
        # lr 0.05 x momentum 0.9 on 12-image tasks is chaotic by the third round (one ReLU-branch flip moves ~10 % of
        # layer4 by 1e-3 - with or without the trained L1 anchor, depending on nothing but rounding); lr 0.01 is not
        OVERRIDES.update(lr=0.01)
    try:
        golden(tmp_path, method, rounds=3, max_factor=25)
    finally:
        OVERRIDES.clear()


def test_fedstil_trained_anchor_under_sgd_matches_reference(tmp_path):
    """``lambda_l1`` large enough (1e-2) for the reference's accidental training of the L1 anchors to be visible under
    SGD as well: with the anchor trained (the default under ``reference_compat``) two rounds agree up to isolated
    ``sign(aw - aw0)`` ties; with a constant anchor more than half of every adaptive tensor is off by ``lr * lambda_l1``
    per step (checked below with the option switched off)."""
    saved = dict(METHOD_OPTS["fedstil"])
    METHOD_OPTS["fedstil"]["lambda_l1"] = 1e-2
    OVERRIDES.update(lr=0.005)
    try:
        golden(tmp_path / "on", "fedstil", max_factor=25)
        with pytest.raises(AssertionError):
            golden(tmp_path / "off", "fedstil", max_factor=25, engine={"train_l1_anchor": False})
    finally:
        METHOD_OPTS["fedstil"] = saved
        OVERRIDES.clear()


@pytest.mark.parametrize("method", ["fedstil", pytest.param("fedavg", marks=full), pytest.param("fedcurv", marks=full)])
def test_world_size_two_matches_reference(tmp_path, method):
    """SURVEY §7.4 "distributed without a cluster": the same experiment with ONE CLIENT PER RANK (gloo, world_size 2;
    the collectives run through ``FedComm``'s gloo emulation of the peer-memory kernels, the server role is replicated)
    against the single-process reference - every file any rank wrote, and every logged metric."""
    import shutil
    splits = _splits()
    ref = _run_reference(tmp_path, method, splits)
    shutil.rmtree(tmp_path / "ref", ignore_errors=True)
    torch.save({"init": ref["init"]}, tmp_path / "ref_out.pt")
    env = dict(os.environ, OMP_NUM_THREADS="4")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--local-addr", "127.0.0.1",
                        "--nproc-per-node", "2", os.path.join(ROOT, "tests", "dist_golden_check.py"), method,
                        str(tmp_path), str(ROUNDS)], env=env, capture_output=True, text=True, timeout=1200)
    assert r.stdout.count("DIST_GOLDEN") == 2, r.stdout[-2000:] + r.stderr[-3000:]
    outs = [torch.load(tmp_path / f"rank{k}_out.pt", weights_only=False) for k in range(2)]
    ignore = FEDCURV_NOT_MATERIALISED if method == "fedcurv" else ()
    bad, seen = [], set()
    for out in outs:
        for name, obj in out["files"].items():
            assert name in ref["files"], f"a rank wrote {name}, the reference did not"
            seen.add(name)
            _compare(name, ref["files"][name], obj, 2e-5, 1e-4, bad, ignore, 25)
    assert not bad, "\n".join(map(str, bad[:20]))
    assert seen == set(ref["files"]), sorted(set(ref["files"]) - seen)
    logged = {}
    for out in outs:
        for client, rounds in (out["log"].get("data") or {}).items():
            logged.setdefault(client, {}).update(rounds)
    for client, rounds in ref["log"]["data"].items():
        for rnd, tasks in rounds.items():
            for task, metrics in tasks.items():
                for k, v in metrics.items():
                    assert abs(float(logged[client][str(rnd)][task][k]) - float(v)) < 1e-3, (client, rnd, task, k)
    for k in range(2):
        shutil.rmtree(tmp_path / f"rank{k}", ignore_errors=True)


def test_early_stopping_matches_reference(tmp_path):
    """Eight epochs at a diverging learning rate: the early-stopping rule (three epochs without a simultaneous loss /
    accuracy improvement, baseline.py:249-255) fires in the fifth epoch, which - as in the reference - is trained but
    not counted (``train_cnt`` = 4 x 12)."""
    OVERRIDES.update(epochs=8, lr=2.0)
    try:
        ref, files = golden(tmp_path, "fedavg", rounds=1)
    finally:
        OVERRIDES.clear()
    assert ref["files"]["client-0/1-client-0-server.ckpt"]["train_cnt"] == 48
    assert files["client-0/1-client-0-server.ckpt"]["train_cnt"] == 48


def test_cross_entropy_plus_triplet_training_matches_reference(tmp_path):
    """``criterion_opts`` as a list: label-smoothing CE + hard-mining triplet loss on the global feature, trained for two
    federated rounds (the reference registers the triplet loss but no shipped config uses it)."""
    OVERRIDES.update(extra_criteria=[{"name": "triplet_loss", "margin": 0.3, "hard_mining": True, "norm_feat": False}])
    try:
        golden(tmp_path, "fedavg")
    finally:
        OVERRIDES.clear()


@pytest.mark.parametrize("method", ["baseline", pytest.param("fedweit", marks=full)])
def test_three_tasks_with_round0_validation_match_reference(tmp_path, method):
    """Per-task checkpoints (``mm`` baseline, FedWeIT) over three tasks, three rounds, with the initial validation pass
    on both sides: a task that was only *validated* must not acquire a checkpoint - the reference's ``load_model`` is a
    no-op without a file, so an untrained task is evaluated with, and trained from, the most recently loaded weights
    (``modules/client.py:63-70``, ``methods/baseline.py:237-238,314-315``)."""
    golden(tmp_path, method, rounds=3, tasks=3, val0=True, max_factor=25)


def test_single_shared_checkpoint_baseline_matches_reference(tmp_path):
    """``baseline`` with ``model_ckpt_name`` set (the reference's "sm" configuration: one model for all tasks)."""
    golden(tmp_path, "baseline+sm_model", rounds=3, max_factor=25)


@full
def test_fedcurv_three_clients_matches_reference(tmp_path):
    """Two *other* clients per penalty: the three pre-reduced moment buffers against the reference's loop over every
    other client's ``(F_j, p_j)`` (fedcurv.py:79-86,621-646), three rounds."""
    golden(tmp_path, "fedcurv", rounds=3, clients=3, max_factor=25, ignore=FEDCURV_NOT_MATERIALISED)


@full
def test_fedavg_with_adam_matches_reference(tmp_path):
    """The reference's shipped optimizer (Adam, lr 1e-3, wd 1e-5), one round. (Adam's first steps turn the *sign* of a
    near-zero gradient into a full +-lr move: in a second round ~0.3 % of the conv weights and a few per cent of the
    512-element BatchNorm biases end ~1e-3 apart - rounding chaos, not arithmetic.)"""
    golden(tmp_path, "fedavg", adam=True, rounds=1, max_factor=150)


def test_fedstil_with_adam_and_trained_anchor_matches_reference(tmp_path):
    """``engine_opts.train_l1_anchor`` (default: on under ``reference_compat``) reproduces the reference optimizer's
    training of FedSTIL's L1 anchors; under Adam that is what makes the first round agree (without it 70-90 % of the
    conv weights differ by ~lr per step).
    One round: from the second on, elements whose loss gradient is ~0 have ``sign(aw - aw0)`` decided by fp32
    rounding order inside the reference itself."""
    golden(tmp_path, "fedstil", adam=True, rounds=1, max_factor=150)


@full
def test_partial_participation_fedavg_matches_reference(tmp_path):
    """``online_clients`` 1 of 2 over four rounds: late first contact, stale uploads in every mean (fedavg.py:386-397)."""
    golden(tmp_path, "fedavg", rounds=4, online=1, max_factor=25)


def test_partial_participation_fedstil_matches_reference(tmp_path):
    """Late first contact receives the server's FedAvg-mean global weight (fedstil.py:1075-1096), the next dispatch is
    a relevance mix over token histories of different lengths. (A few ReLU-branch flips are larger here - the heads are
    far from converged, gradients are big - hence the wider bound on isolated elements. lr 0.01 for the same reason as
    the three-round test: with the trained L1 anchor the lr-0.05 momentum trajectory amplifies one flip into a
    visibly different third round.)"""
    OVERRIDES.update(lr=0.01)
    try:
        golden(tmp_path, "fedstil", rounds=3, online=1, max_factor=100)
    finally:
        OVERRIDES.clear()


@full
def test_fedstil_on_resnet50_first_round_matches_reference(tmp_path):
    """The headline backbone (``configs/backbone/experiment_fedstil_res50.yaml``): bottleneck blocks, eleven adaptive
    layers, 1024-channel prototypes. One round - with nine ReLUs per sample position in ``layer4`` the branch flips
    of a second round already touch ~5 % of the conv weights (by <= 6e-4)."""
    golden(tmp_path, "fedstil@resnet50", rounds=1)


def test_fedstil_on_swin_matches_reference(tmp_path):
    """FedSTIL over Swin-T (``configs/backbone/experiment_fedstil_swin.yaml``: ``base.layers.3`` + classifier, nine
    adaptive layers with biases, LayerNorm / relative-position tables trained locally, 49 x 768 token maps)."""
    golden(tmp_path, "fedstil@swin_transformer_tiny")


def test_icarl_first_round_matches_reference(tmp_path):
    """One round only: from the second round on the reference distils every exemplar towards the recorded logits of a
    *random* exemplar (two independent DataLoader shuffles, icarl.py:86-95,219-223), which no seed alignment can
    reproduce bit for bit; the first round covers training, herding, the grown head and the checkpoint schema."""
    golden(tmp_path, "icarl", rounds=1)

"""Byzantine-robust aggregation of the FedAvg family (``server: aggregator:``; coordinate-wise median and trimmed mean).

A float64 oracle built from the definition (checked against hand-computed cases, ``numpy.median`` and
``scipy.stats.trim_mean``), the CPU path and ``fed_reduce_robust_kernel`` under the SIMT emulator's multi-rank mode
against it, configuration refusals, and tiny FedAvg / FedProx / FedCurv experiments with one Byzantine client.

Definition: per coordinate the K values are ordered by ``(value, position in the client list)`` - NaN above +inf,
-0.0 == +0.0 broken by position - i.e. a stable sort. ``median``: the middle value for odd K, ``0.5f * lo + 0.5f * hi``
in fp32 for even K. ``trimmed_mean``: the mean of sorted positions ``[b, K - b)``, ``b = floor(beta * K)``.

Bounds: medians are bitwise equal to the oracle (for normal-range inputs the float64 midpoint rounded to fp32 is the
fp32 expression exactly: both halves are exact and the sum is rounded once). A trimmed mean summed in fp32 in ascending
order is within ``(K - 2b) * 2^-23 * max|kept|`` of the float64 mean."""
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

NAN, INF = float("nan"), float("inf")


# ---------------------------------------------------------------------------------------------------------- oracle
def oracle(vals, rule, b=0):
    """``vals``: ``[K, n]`` fp32 (tensor, any device). Returns the float64 aggregate (the even-K median is the fp32
    midpoint, which the float64 one rounds to exactly)."""
    v = torch.as_tensor(vals, dtype=torch.float32).double()
    K = v.shape[0]
    s = torch.sort(v, dim=0, stable=True).values
    if rule == "median":
        if K % 2:
            return s[(K - 1) // 2]
        return 0.5 * s[K // 2 - 1] + 0.5 * s[K // 2]
    return s[b:K - b].sum(0) / (K - 2 * b)


def trimmed_bound(vals, b):
    """``(K - 2b) * 2^-23 * max|kept|`` per coordinate (float64)."""
    s = torch.sort(torch.as_tensor(vals, dtype=torch.float32).double(), dim=0, stable=True).values
    K = s.shape[0]
    return (K - 2 * b) * 2.0 ** -23 * s[b:K - b].abs().max(0).values


def check_against_oracle(got, vals, rule, b=0):
    ref = oracle(vals, rule, b)
    got = got.detach().cpu()
    if rule == "median":
        # bitwise wherever the oracle is a number; NaN where it is NaN (the payload of a NaN formed by the even-K
        # midpoint depends on the hardware)
        want = ref.float().cpu()
        nan = torch.isnan(want)
        assert torch.equal(torch.isnan(got), nan)
        assert torch.equal(got[~nan].view(torch.int32), want[~nan].view(torch.int32)), \
            float((got[~nan].double() - ref.cpu()[~nan]).abs().max())
    else:
        err = (got.double() - ref.cpu()).abs() - trimmed_bound(vals, b).cpu()
        assert bool((err <= 0).all()), float(err.max())


def bits(x):
    return np.float32(x).view(np.uint32)


def col(*xs):
    return torch.tensor(xs, dtype=torch.float32)[:, None]


def test_oracle_hand_computed_medians():
    assert float(oracle(col(3, 1, 2), "median")) == 2.0
    assert float(oracle(col(4, 1, 3, 2), "median")) == 2.5
    assert float(oracle(col(7), "median")) == 7.0
    # ties: (value, position) order - equal values keep their positions
    assert float(oracle(col(2, 2, 1, 2), "median")) == 2.0
    # +-0 compare equal and the tie goes to the lower position
    assert bits(float(oracle(col(0.0, -0.0, 1), "median"))) == bits(-0.0)
    assert bits(float(oracle(col(-0.0, 0.0, 1), "median"))) == bits(0.0)
    assert bits(float(oracle(col(-0.0, -1, 0.0), "median"))) == bits(-0.0)
    # infinities
    assert float(oracle(col(INF, -INF, 5), "median")) == 5.0
    assert float(oracle(col(INF, 1), "median")) == INF
    assert math.isnan(float(oracle(col(INF, -INF), "median")))
    # NaN sorts above +inf
    assert float(oracle(col(NAN, 1, 2), "median")) == 2.0
    assert float(oracle(col(NAN, INF, 1), "median")) == INF
    assert float(oracle(col(NAN, 3, 1, 2), "median")) == 2.5
    assert math.isnan(float(oracle(col(NAN, NAN, 1), "median")))
    # the midpoint cannot overflow
    assert float(oracle(col(3e38, 3e38), "median")) == float(np.float32(3e38))


def test_oracle_hand_computed_trimmed_means():
    assert float(oracle(col(5, 1, 4, 2, 3), "trimmed_mean", 0)) == 3.0
    assert float(oracle(col(5, 1, 4, 2, 3), "trimmed_mean", 1)) == 3.0      # (2 + 3 + 4) / 3
    assert float(oracle(col(5, 1, 4, 2, 3), "trimmed_mean", 2)) == 3.0      # b at its maximum: the middle value
    assert float(oracle(col(10, 1, 2, 3, -100), "trimmed_mean", 1)) == 2.0
    assert float(oracle(col(NAN, 1, 2, 3, 4), "trimmed_mean", 1)) == 3.0    # NaN is the largest value: cut
    assert float(oracle(col(-INF, 1, 2, 6, INF), "trimmed_mean", 1)) == 3.0
    assert float(oracle(col(1, 2, 4, 100), "trimmed_mean", 1)) == 3.0       # b at its maximum for even K
    assert math.isnan(float(oracle(col(NAN, 1), "trimmed_mean", 0)))
    from flpr_b200.methods.fedbase import trim_count
    assert trim_count(0.2, 2) == 0 and trim_count(0.2, 10) == 2 and trim_count(0.1, 30) == 3
    assert trim_count(0.49, 32) == 15 and trim_count(0.0, 32) == 0 and trim_count(0.25, 3) == 0


@pytest.mark.parametrize("K", [1, 2, 3, 4, 7, 8, 31, 32])
def test_oracle_agrees_with_numpy_and_scipy(K):
    from scipy import stats
    from flpr_b200.methods.fedbase import trim_count
    g = torch.Generator().manual_seed(K)
    vals = torch.randn(K, 2000, generator=g) * torch.exp(2 * torch.randn(K, 2000, generator=g))
    med = oracle(vals, "median").float().numpy()
    ref = np.median(vals.numpy().astype(np.float64), axis=0).astype(np.float32)
    ulp = np.spacing(np.abs(ref).astype(np.float32))
    assert (np.abs(med.astype(np.float64) - ref) <= ulp).all()
    for beta in (0.0, 0.1, 0.2, 0.25, 0.49):
        b = trim_count(beta, K)
        tm = oracle(vals, "trimmed_mean", b).numpy()
        ref = stats.trim_mean(vals.numpy().astype(np.float64), beta, axis=0)
        assert (np.abs(tm - ref) <= trimmed_bound(vals, b).numpy()).all(), beta


# ---------------------------------------------------------------------------------------------------------- CPU path
def special_values(K, n, seed):
    """Normal-range random values with ties, signed zeros, infinities and NaN mixed in."""
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(K, n, generator=g)
    v[:, ::7] = torch.randint(-2, 3, (K, len(range(0, n, 7))), generator=g).float()          # ties
    v[:, 1::11] = torch.where(torch.rand(K, len(range(1, n, 11)), generator=g) < 0.5, 0.0, -0.0)  # signed zeros
    v[0, 2::13] = INF
    v[-1, 3::17] = -INF
    v[K // 2, 5::19] = NAN
    return v


@pytest.mark.parametrize("K", [1, 2, 3, 4, 5, 8, 17, 32])
def test_cpu_path_matches_oracle(K):
    from flpr_b200.parallel.comm import FedComm
    n = 4 * 257
    comm = FedComm("cpu", K, arena_bytes=(K + 1) * n * 4 + (1 << 16))
    comm.alloc_client_buffer("up", n)
    comm.alloc_rank_buffer("glob", n)
    vals = special_values(K, n, K)
    for c in range(K):
        comm.client_view("up", c).copy_(vals[c])
    order = list(range(K))[::-1]                       # the position is the position in the client list
    comm.reduce_robust("up", "glob", order, "median")
    assert torch.equal(comm.rank_view("glob").view(torch.int32), oracle(vals[order], "median").float().view(torch.int32))
    for b in sorted({0, (K - 1) // 2}):
        comm.reduce_robust("up", "glob", order, "trimmed_mean", b)
        finite = torch.isfinite(vals).all(0)
        check_against_oracle(comm.rank_view("glob")[finite], vals[order][:, finite], "trimmed_mean", b)
    with pytest.raises(ValueError):
        comm.reduce_robust("up", "glob", order, "trimmed_mean", (K + 1) // 2 if K > 1 else 1)
    with pytest.raises(ValueError):
        comm.reduce_robust("up", "glob", order, "mode")


# ---------------------------------------------------------------------------------------------------------- emulated kernel
@pytest.fixture(scope="module")
def lib():
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    from emu import comm_harness as H
    from emu.build_emu import build
    from flpr_b200.ops import native
    try:
        handle = H.load(build("fedcomm.cu"))
    except RuntimeError as ex:
        pytest.skip(f"emulator build unavailable: {ex}")
    native.declare_present(handle)
    yield handle
    assert handle.flpr_emu_deadlocks() == 0


def _run(lib, seed):
    from emu import comm_harness as H
    assert H.run(lib, seed) == 0


def _done(lib):
    from emu import comm_harness as H
    H.end(lib)


def normal_values(K, n, seed):
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(K, n, generator=g) * torch.exp(torch.randn(K, n, generator=g))
    v[:, ::5] = torch.randint(-1, 2, (K, len(range(0, n, 5))), generator=g).float()        # ties and +-0
    v[:, ::9] = -v[:, ::9]
    return v


_SCHEDULES = [
    # world, number of clients, participants, n
    (1, 1, [0], 4),
    (1, 3, [2, 0, 1], 4 * 300),
    (2, 2, [1, 0], 4 * 513),
    (2, 5, [4, 1, 3], 8),
    (3, 6, [0, 3], 4 * 700),                 # ranks 1 and 2 host no participant
    (3, 7, [6, 5, 4, 3, 2, 1, 0], 4 * 5),
    (8, 32, list(range(32)), 4 * 520),        # a few grid strides per rank's slice
    (8, 32, list(range(31, -1, -1)), 12),
    (8, 9, [8, 0], 4 * 64),                   # six of eight ranks host none
]


@pytest.mark.parametrize("world,clients,part,n", _SCHEDULES)
def test_emulated_kernel_matches_oracle_on_every_rank(lib, world, clients, part, n):
    """``FedComm.reduce_robust`` in ``p2p`` mode on ``world`` emulated ranks, under seeded random schedules: medians
    bitwise equal to the oracle, trimmed means within the bound, every rank's ``dst`` bitwise identical."""
    from emu import comm_harness as H
    from flpr_b200.methods.fedbase import trim_count
    comms = H.make_fedcomm_world(lib, world, clients, arena_bytes=(clients + world) * n * 4 + (1 << 20), blocks=2)
    for c in comms:
        c.alloc_client_buffer("up", n)
        c.alloc_rank_buffer("glob", n)
    vals = normal_values(clients, n, 100 * world + clients)
    for c in comms:
        for cid in c.local_clients():
            c.client_view("up", cid).copy_(vals[cid])
    K = len(part)
    cases = [("median", 0), ("trimmed_mean", 0), ("trimmed_mean", trim_count(0.2, K)),
             ("trimmed_mean", (K - 1) // 2)]
    for seed, (rule, b) in enumerate(cases):
        for c in comms:
            c.glob_before = c.bytes_moved
            c.reduce_robust("up", "glob", part, rule, b)
            assert c.nvls_launches == 0
        _run(lib, 7 * seed + world)
        for c in comms:
            assert c.error_word() == 0
            assert torch.equal(c.rank_view("glob").view(torch.int32), comms[0].rank_view("glob").view(torch.int32))
            if world > 1:
                assert c.bytes_moved > c.glob_before
        check_against_oracle(comms[0].rank_view("glob"), vals[part], rule, b)
    _done(lib)


def test_emulated_kernel_return_codes(lib):
    from emu import comm_harness as H
    w = H.EmuWorld(lib, 1)
    src, dst = [torch.zeros(8) for _ in range(3)], [torch.zeros(8)]
    S, D = H.ptr_array(src), H.ptr_array(dst)

    def call(K, rule, b, n=8, world=1):
        return lib.flpr_comm_reduce_robust(0, world, w._pages, 1.0, K, S, D, rule, b, n, 1, w.stream(0))
    assert call(0, 0, 0) == -1 and call(33, 0, 0) == -1 and call(3, 0, 0, world=9) == -1
    assert call(3, 0, 0, n=6) == -2
    assert call(3, 2, 0) == -3 and call(3, -1, 0) == -3            # unknown rule
    assert call(3, 0, 1) == -3                                     # the median takes no b
    assert call(3, 1, 2) == -3 and call(3, 1, -1) == -3 and call(2, 1, 1) == -3
    assert call(3, 1, 1) == 0 and call(3, 0, 0) == 0
    _run(lib, 1)
    w.close()


def test_emulated_back_to_back_rounds_read_nothing_early_or_stale(lib):
    """Every rank queues: robust aggregate of round A, archive of the result, its clients' round-B uploads, robust
    aggregate of round B, archive - all device-ordered on its stream, nothing host-synchronised in between. Both
    archives must be their round's aggregate exactly: a kernel that read an upload before its owner rewrote it, or
    pushed into a ``dst`` a rank was still archiving, would show."""
    from emu import comm_harness as H
    world, K, n = 3, 5, 4 * 300
    w = H.EmuWorld(lib, world, blocks=3)
    A, B = normal_values(K, n, 1), normal_values(K, n, 2)
    up = [A[c].clone() for c in range(K)]
    nxt = [B[c].clone() for c in range(K)]
    glob = [torch.full((n,), -1.0) for _ in range(world)]
    arch = [[torch.zeros(n) for _ in range(world)] for _ in range(2)]
    order = [3, 0, 4, 1, 2]

    def robust(r, rule, b):
        rc = lib.flpr_comm_reduce_robust(r, world, w._pages, w.timeout_s, K, H.ptr_array([up[c] for c in order]),
                                         H.ptr_array(glob), rule, b, n, w.blocks, w.stream(r))
        assert rc == 0
    for r in range(world):
        robust(r, 0, 0)
        w.local_copy(r, glob[r], arch[0][r])
        for c in range(K):
            if c % world == r:
                w.local_copy(r, nxt[c], up[c])
        robust(r, 1, 1)
        w.local_copy(r, glob[r], arch[1][r])
    assert w.run(11) == 0
    for r in range(world):
        assert torch.equal(arch[0][r], oracle(A[order], "median").float())
        check_against_oracle(arch[1][r], B[order], "trimmed_mean", 1)
        assert torch.equal(arch[1][r], arch[1][0])
        assert w.error_word(r) == 0
    w.close()


def test_emulated_missing_rank_trips_the_watchdog_and_publishes_nothing(lib):
    from emu import comm_harness as H
    from flpr_b200.ops.native import NativeError
    world, clients, n = 3, 6, 4 * 100
    comms = H.make_fedcomm_world(lib, world, clients, timeout_s=2e-4)
    for c in comms:
        c.alloc_client_buffer("up", n)
        c.alloc_rank_buffer("glob", n)
        for cid in c.local_clients():
            c.client_view("up", cid).copy_(torch.randn(n))
        c.rank_view("glob").fill_(-1.0)
    for c in comms[:2]:
        c.reduce_robust("up", "glob", list(range(clients)), "median")
        c.poll_errors()
    _run(lib, 2)
    for c in comms[:2]:
        with pytest.raises(NativeError, match="timed out waiting for a peer rank"):
            c.poll_errors()
    for c in comms:
        assert bool((c.rank_view("glob") == -1.0).all())
    comms[2].poll_errors()
    _done(lib)


# ---------------------------------------------------------------------------------------------------------- configuration
@pytest.mark.parametrize("bad", [
    {"name": "mean"}, {}, {"beta": 0.1}, {"name": "median", "beta": 0.1}, {"name": "trimmed_mean", "alpha": 0.1},
    {"name": "trimmed_mean", "beta": 0.5}, {"name": "trimmed_mean", "beta": -0.01}, {"name": "trimmed_mean", "beta": 1},
    {"name": "trimmed_mean", "beta": NAN}, {"name": "trimmed_mean", "beta": INF}, {"name": "trimmed_mean", "beta": "0.1"},
    {"name": "trimmed_mean", "beta": None}, {"name": "trimmed_mean", "beta": True}, "median", ["median"]])
def test_bad_aggregator_is_refused(bad):
    from flpr_b200.methods.fedbase import parse_aggregator
    with pytest.raises(ValueError):
        parse_aggregator(bad)


def test_aggregator_defaults():
    from flpr_b200.methods.fedbase import parse_aggregator
    assert parse_aggregator(None) is None
    assert parse_aggregator({"name": "median"}) == {"name": "median"}
    assert parse_aggregator({"name": "trimmed_mean"}) == {"name": "trimmed_mean", "beta": 0.1}
    assert parse_aggregator({"name": "trimmed_mean", "beta": 0}) == {"name": "trimmed_mean", "beta": 0.0}


def test_bad_aggregator_fails_at_server_construction(tmp_path):
    from flpr_b200.runtime.builder import parser_server
    common = tiny_common(str(tmp_path))
    cfg = tiny_experiment(common, "fedprox")
    cfg["server"]["aggregator"] = {"name": "trimmed_mean", "beta": 0.5}
    with pytest.raises(ValueError, match="beta"):
        parser_server(cfg, common)


@pytest.mark.parametrize("method", ["fedstil", "fedstil-atten", "fedweit", "ewc", "mas", "si", "icarl", "baseline"])
def test_aggregator_refused_for_methods_without_a_fedavg_server(tmp_path, method):
    from flpr_b200.runtime.builder import parser_server
    common = tiny_common(str(tmp_path))
    cfg = tiny_experiment(common, method)
    cfg["server"]["aggregator"] = {"name": "median"}
    with pytest.raises(ValueError, match="aggregator"):
        parser_server(cfg, common)


# ---------------------------------------------------------------------------------------------------------- experiments
BYZANTINE = "client-0"


def poison_uploads(monkeypatch):
    """After its upload, client-0's slot holds 1e30 and NaN in alternating thirds of the coordinates (the payload
    checkpoint records the poisoned values: it is written from views of the slot)."""
    from flpr_b200.methods.fedbase import FedClient
    inner = FedClient.get_incremental_state

    def poisoned(self, **kw):
        st = inner(self, **kw)
        if self.client_name == BYZANTINE:
            slot = self.comm.client_view("up", self.client_id)
            slot[0::3] = 1e30
            slot[1::3] = NAN
        return st
    monkeypatch.setattr(FedClient, "get_incremental_state", poisoned)


def run_experiment(tmp, method="fedavg", aggregator=None, server_opt=None, rounds=3, n_clients=4, online=None,
                   device="cpu", factory=None, **task_over):
    common = tiny_common(str(tmp), device=device)
    common["defaults"]["exp_opts"]["comm_rounds"] = rounds
    common["defaults"]["exp_opts"]["online_clients"] = online or n_clients
    for key, val in task_over.items():
        common["defaults"]["task_opts"][key].update(val)
    cfg = tiny_experiment(common, method, n_clients=n_clients)
    if aggregator is not None:
        cfg["server"]["aggregator"] = dict(aggregator)
    if server_opt is not None:
        cfg["server"]["server_opt"] = dict(server_opt)
    with ExperimentStage(common, [cfg], source_factory=factory or tiny_factory()) as stage:
        log = stage.run_experiment(cfg)
    return os.path.join(common["checkpoints_dir"], cfg["exp_name"]), log


def _load(root, actor, name):
    path = os.path.join(root, actor, f"{name}.ckpt")
    return torch.load(path, weights_only=False) if os.path.exists(path) else None


def _payload(st):
    return st.get("incremental_model_params") or st.get("integrated_model_params")


def replay_dispatches(root, aggregator, rounds, n_clients):
    """Recompute in float64 the aggregate of every round from the upload checkpoints (offline clients keep their last
    upload) and compare it with every dispatch of the next round. Returns the number of dispatches compared."""
    from flpr_b200.methods.fedbase import trim_count
    names = [f"client-{i}" for i in range(n_clients)]
    latest = {}
    checked = 0
    for r in range(1, rounds):
        for n in names:
            up = _load(root, n, f"{r}-{n}-server")
            if up is not None:
                latest[n] = up["incremental_model_params"]
        keys = sorted(next(iter(latest.values())))
        stack = torch.stack([torch.cat([latest[n][k].float().flatten() for k in keys]) for n in sorted(latest)])
        b = trim_count(aggregator.get("beta", 0.1), len(latest)) if aggregator["name"] == "trimmed_mean" else 0
        ref = oracle(stack, aggregator["name"], b)
        if aggregator["name"] == "median":
            ref = ref.float().double()                 # (the fp32 median, which the float64 one rounds to)
        tol = trimmed_bound(stack, b) if aggregator["name"] == "trimmed_mean" else torch.zeros_like(ref)
        for n in names:
            st = _load(root, "server", f"{r + 1}-server-{n}")
            if st is None:
                continue
            got = torch.cat([_payload(st)[k].double().flatten() for k in keys])
            assert bool(torch.isfinite(got).all()), f"round {r + 1} dispatch to {n} is not finite"
            assert bool(((got - ref).abs() <= tol).all()), f"round {r + 1} dispatch to {n}"
            checked += 1
    return checked


@pytest.mark.parametrize("method,aggregator", [("fedavg", {"name": "median"}),
                                               ("fedprox", {"name": "trimmed_mean", "beta": 0.25}),
                                               ("fedcurv", {"name": "median"})])
def test_byzantine_client_is_outvoted(tmp_path, monkeypatch, method, aggregator):
    """Four clients, all online; client-0 uploads 1e30 / NaN. The replica stays finite and every dispatch is the
    float64 replay of the aggregator over that round's upload checkpoints. FedCurv runs two rounds: its curvature
    moments are sums over every upload, so the poisoned parameters reach the honest clients' penalty and their next
    uploads - the aggregator protects the replica, not the curvature exchange."""
    poison_uploads(monkeypatch)
    rounds = 2 if method == "fedcurv" else 3
    root, _ = run_experiment(tmp_path, method, aggregator=aggregator, rounds=rounds, n_clients=4)
    up = _load(root, BYZANTINE, f"1-{BYZANTINE}-server")["incremental_model_params"]
    assert any(bool(torch.isnan(t).any()) for t in up.values()), "the poisoned upload was not checkpointed"
    assert replay_dispatches(root, aggregator, rounds, 4) >= 4 * (rounds - 1)


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


def _key_tree(obj):
    if isinstance(obj, dict):
        return {k: _key_tree(val) for k, val in obj.items()}
    return type(obj).__name__ if not torch.is_tensor(obj) else ("tensor", tuple(obj.shape))


def _tensors(obj, prefix=""):
    if torch.is_tensor(obj):
        return {prefix: obj}
    if isinstance(obj, dict):
        out = {}
        for k, val in obj.items():
            out.update(_tensors(val, f"{prefix}/{k}"))
        return out
    return {}


@pytest.mark.parametrize("method", ["fedavg", "fedcurv"])
def test_checkpoint_and_payload_schemas_unchanged(tmp_path, method):
    root_a, _ = run_experiment(tmp_path / "plain", method, rounds=2, n_clients=3)
    root_b, _ = run_experiment(tmp_path / "median", method, aggregator={"name": "median"}, rounds=2, n_clients=3)
    fa, fb = _model_files(root_a), _model_files(root_b)
    assert set(fa) == set(fb) and any("-server-" in f for f in fa)
    for f in fa:
        assert _key_tree(fa[f]) == _key_tree(fb[f]), f
    moved = [f for f in fa if f.startswith("server/2-")]
    assert moved and any(not torch.equal(_tensors(fa[f])[k], _tensors(fb[f])[k]) for f in moved
                         for k in _tensors(fa[f])), "the aggregator did not change the dispatch"


def test_trimmed_mean_without_trimming_is_fedavg_with_equal_counts(tmp_path):
    """``beta: 0`` and equal ``train_cnt`` (every client trains on the same number of images): the first dispatch that
    follows an aggregation (round 2) equals plain FedAvg's within fp32 reordering."""
    root_a, _ = run_experiment(tmp_path / "plain", n_clients=3)
    root_b, _ = run_experiment(tmp_path / "tm0", aggregator={"name": "trimmed_mean", "beta": 0}, n_clients=3)
    cnts = {float(_load(root_a, f"client-{i}", f"1-client-{i}-server")["train_cnt"]) for i in range(3)}
    assert len(cnts) == 1, cnts
    fa, fb = _model_files(root_a), _model_files(root_b)
    second = [f for f in fa if f.startswith("server/2-")]
    assert second
    for f in second:
        ta, tb = _tensors(fa[f]), _tensors(fb[f])
        assert set(ta) == set(tb)
        for k in ta:
            a, b = ta[k].double(), tb[k].double()
            assert torch.allclose(a, b, rtol=1e-6, atol=1e-6 * float(a.abs().max()) + 1e-12), (f, k)


def test_composes_with_server_opt(tmp_path):
    """``server_opt: sgd, lr 1`` steps the replica all the way to the robust aggregate: the dispatches are the replay
    of the median (within the step's own rounding); with ``adam`` the replica moves toward it and stays finite."""
    from test_server_opt import oracle_step
    root, _ = run_experiment(tmp_path / "sgd", aggregator={"name": "median"}, server_opt={"name": "sgd", "lr": 1.0},
                             n_clients=3)
    names = [f"client-{i}" for i in range(3)]
    latest = {}
    for r in (1, 2):
        for n in names:
            up = _load(root, n, f"{r}-{n}-server")
            if up is not None:
                latest[n] = up["incremental_model_params"]
        keys = sorted(next(iter(latest.values())))
        med = oracle(torch.stack([torch.cat([latest[n][k].float().flatten() for k in keys]) for n in sorted(latest)]),
                     "median")
        prev = torch.cat([_payload(_load(root, "server", f"{r}-server-{names[0]}"))[k].double().flatten()
                          for k in keys])
        x, _, _, _ = oracle_step("sgd", prev.numpy(), med.numpy(), np.zeros(len(prev)), None, lr=1.0)
        got = torch.cat([_payload(_load(root, "server", f"{r + 1}-server-{names[0]}"))[k].double().flatten()
                         for k in keys])
        np.testing.assert_allclose(got.numpy(), x, rtol=1e-6, atol=1e-6 * float(np.abs(x).max()))
    root, _ = run_experiment(tmp_path / "adam", aggregator={"name": "trimmed_mean", "beta": 0.25},
                             server_opt={"name": "adam", "lr": 0.01}, n_clients=4)
    got = _payload(_load(root, "server", "3-server-client-1"))
    assert all(bool(torch.isfinite(t).all()) for t in got.values())


# ---------------------------------------------------------------------------------------------------------- two ranks
def test_gloo_two_ranks_keep_identical_replicas(tmp_path):
    """World size 2 on gloo, median over three clients with client-0 Byzantine: replicas bit-identical across ranks
    and equal to the float64 replay of the median over the uploads both ranks checkpointed."""
    script = os.path.join(os.path.dirname(__file__), "dist_robust_agg_check.py")
    env = dict(os.environ, FLPR_TMP=str(tmp_path), OMP_NUM_THREADS="2")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--local-addr", "127.0.0.1",
                        "--nproc-per-node", "2", script, "cpu"], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "DIST_ROBUST_AGG OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]

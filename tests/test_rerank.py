"""k-reciprocal re-ranking (``ops/rank.py``, ``csrc/rerank.cu``) in the CPU tier: the float64 reference against a case
worked out by hand, parameter checks, every kernel stage under the SIMT emulator of ``tests/emu`` against the reference's
intermediates on the same ``D``, and the engine option ``engine_opts.re_ranking``."""
import math
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch


# ------------------------------------------------------------------------------------------------------------ reference
def test_reference_on_a_case_checked_by_hand():
    """Six points on a line, two well separated groups {0, 1, 2} / {10, 11, 13}; k1 = 2 (K = 3 neighbours with the
    point itself), h = round(1) + 1 = 2, k2 = 1 (no query expansion), lambda = 0.3.

    x = [0, 10 | 1, 2, 11, 13]  (two queries, four gallery items).  First three neighbours by squared distance:
        R0 = [0, 2, 3]   R1 = [1, 4, 5]   R2 = [2, 0, 3] (0 and 3 tie at 1: the lower index first)
        R3 = [3, 2, 0]   R4 = [4, 1, 5]   R5 = [5, 4, 1]
    Every neighbour lists its point back, so K(i) = R_i. Expansion of row 0: c = 0 -> {0, 2}, c = 2 -> {2, 0}, c = 3 ->
    {3} (3 is not in R2[:2] = [2, 0]); all three pass the 2/3 test, so E(0) = {0, 2, 3}; likewise E(1) = {1, 4, 5}."""
    from flpr_b200.ops.rank import re_ranking, re_ranking_reference
    q = torch.tensor([[0.0], [10.0]])
    g = torch.tensor([[1.0], [2.0], [11.0], [13.0]])
    final, det = re_ranking_reference(q, g, k1=2, k2=1, lambda_value=0.3, details=True)
    assert det["R"].tolist() == [[0, 2, 3], [1, 4, 5], [2, 0, 3], [3, 2, 0], [4, 1, 5], [5, 4, 1]]
    assert det["K"] == [[0, 2, 3], [1, 4, 5], [2, 0, 3], [3, 2, 0], [4, 1, 5], [5, 4, 1]]
    assert [e.tolist() for e in det["E"]] == [[0, 2, 3], [1, 4, 5], [0, 2, 3], [0, 2, 3], [1, 4, 5], [1, 4, 5]]

    # rows of D divided by their maxima: 169 (x = 0, 13), 144 (x = 1), 121 (x = 2, 11), 100 (x = 10)
    def w(ds):                                     # V over E: exp(-d) / sum
        e = [math.exp(-d) for d in ds]
        return [v / sum(e) for v in e]
    V = {0: w([0, 1 / 169, 4 / 169]), 2: w([1 / 144, 0, 1 / 144]), 3: w([4 / 121, 1 / 121, 0]),
         1: w([0, 1 / 100, 9 / 100]), 4: w([1 / 121, 0, 4 / 121]), 5: w([9 / 169, 4 / 169, 0])}
    assert np.allclose(det["V"][0, [0, 2, 3]], V[0], rtol=0, atol=1e-15)

    def jac(a, b):
        m = sum(min(x, y) for x, y in zip(V[a], V[b]))
        return 1 - m / (2 - m)
    expected = [[0.7 * jac(0, 2) + 0.3 * 1 / 169, 0.7 * jac(0, 3) + 0.3 * 4 / 169, 0.7 + 0.3 * 121 / 169,
                 0.7 + 0.3 * 169 / 169],
                [0.7 + 0.3 * 81 / 100, 0.7 + 0.3 * 64 / 100, 0.7 * jac(1, 4) + 0.3 * 1 / 100,
                 0.7 * jac(1, 5) + 0.3 * 9 / 100]]
    assert torch.allclose(final, torch.tensor(expected, dtype=torch.float64), rtol=0, atol=1e-12)
    out = re_ranking(q, g, k1=2, k2=1, lambda_value=0.3)             # CPU tensors: the reference, as fp32
    assert out.dtype == torch.float32 and torch.equal(out, final.float())


@pytest.mark.parametrize("k1,k2,lam", [(0, 1, 0.3), (64, 6, 0.3), (20, 0, 0.3), (20, 22, 0.3), (20, 6, -0.1),
                                       (20, 6, 1.5), (20.0, 6, 0.3), (True, 1, 0.3), (20, 6, "0.3")])
def test_re_ranking_rejects_bad_parameters(k1, k2, lam):
    from flpr_b200.ops.rank import re_ranking
    q, g = torch.randn(3, 4), torch.randn(5, 4)
    with pytest.raises(ValueError):
        re_ranking(q, g, k1=k1, k2=k2, lambda_value=lam)


def test_re_ranking_option_values():
    from flpr_b200.ops.rank import re_ranking_params
    assert re_ranking_params(False) is None and re_ranking_params(None) is None
    assert re_ranking_params(True) == {"k1": 20, "k2": 6, "lambda_value": 0.3}
    assert re_ranking_params({"k1": 10, "lambda_value": 0}) == {"k1": 10, "k2": 6, "lambda_value": 0.0}
    for bad in ({"k3": 1}, "yes", 1, {"k1": 5, "k2": 7}):
        with pytest.raises(ValueError):
            re_ranking_params(bad)


def test_evaluate_with_re_ranking_on_cpu():
    """``evaluate(..., re_ranking=...)`` ranks by the negated reference distance; ``None`` is the plain path."""
    from flpr_b200.data.synthetic import clustered_features
    from flpr_b200.ops.rank import evaluate, rank_metrics_reference, re_ranking_reference, similarity
    q, ql, g, gl = clustered_features(12, 60, 16, 8, seed=3)
    cmc, m_ap = evaluate(q, ql, g, gl, re_ranking={"k1": 6, "k2": 3})
    ref_cmc, ref_map = rank_metrics_reference(-re_ranking_reference(q, g, 6, 3, 0.3).float(), ql, gl)
    assert np.array_equal(cmc, ref_cmc) and m_ap == ref_map
    plain = evaluate(q, ql, g, gl)
    base = rank_metrics_reference(similarity(q, g), ql, gl)
    assert np.array_equal(plain[0], base[0]) and plain[1] == base[1]


# ------------------------------------------------------------------------------------------------------------ emulator
@pytest.fixture(scope="module")
def emu_rerank():
    if shutil.which("g++") is None:
        pytest.skip("g++ not available")
    from emu.build_emu import build
    try:
        return build("rerank.cu")
    except RuntimeError as ex:
        pytest.skip(f"emulator build unavailable: {ex}")


def _dense(sp, n):
    return sp.dense(n).numpy()


@pytest.mark.parametrize("nq,ng,k1,k2,lam,tile", [
    (7, 30, 50, 6, 0.3, 0),        # N < k1 + 1: every range clamps to N
    (20, 90, 20, 6, 0.3, 16),      # the gallery spans six shared-memory tiles
    (15, 60, 10, 1, 0.0, 0),       # k2 = 1: no query expansion; lambda = 0
    (9, 41, 4, 5, 1.0, 0),         # duplicated features: tied distances; lambda = 1
])
def test_kernel_stages_match_the_reference_under_the_emulator(emu_rerank, nq, ng, k1, k2, lam, tile):
    from flpr_b200.data.synthetic import clustered_features
    from flpr_b200.ops import native, rank
    q, _, g, _ = clustered_features(nq, ng, 24, max(3, (nq + ng) // 8), seed=nq)
    if lam == 1.0:
        g[3] = g[2]
        g[7] = q[0]
    n = nq + ng
    native.use_emulated_libraries([emu_rerank])
    try:
        before = native.launches()
        x = torch.cat([q, g]).float()
        D = rank.rr_distance(rank.similarity(x, x), x)
        R = rank.rr_topk(D, k1)
        V = rank.rr_encode(D, R, k1)
        Vq = rank.rr_expand(V, R, k2)
        out = rank.rr_jaccard(Vq, D, nq, lam, tile)
        whole = rank.re_ranking(q, g, k1, k2, lam)               # the public entry, same kernels
        assert native.launches() > before
    finally:
        native.use_emulated_libraries(None)
    assert (D.double() - rank.re_ranking_distance_reference(q, g)).abs().max() < 1e-6
    ref, det = rank.re_ranking_reference(q, g, k1, k2, lam, distance=D, details=True)
    assert R.shape == (n, min(k1 + 1, n)) and np.array_equal(R.numpy(), det["R"])
    assert np.abs(_dense(V, n) - det["V"]).max() < 1e-6
    assert np.abs(_dense(Vq, n) - det["Vq"]).max() < 1e-6
    for i in range(n):                                           # sparse rows: ascending, no duplicates
        c = V.cols[i, :V.nnz[i]].tolist()
        assert c == sorted(set(c)) == det["E"][i].tolist()
    assert out.shape == (nq, ng) and (out.double() - ref).abs().max() < 1e-5
    assert torch.equal(whole, out)


def test_row_wise_reference_matches_the_whole_reference():
    from flpr_b200.data.synthetic import clustered_features
    from flpr_b200.ops import rank
    q, _, g, _ = clustered_features(10, 50, 16, 6, seed=1)
    _, det = rank.re_ranking_reference(q, g, 8, 3, 0.3, details=True)
    R = rank.re_ranking_topk_reference(det["D"], 8, rows=[4, 17])
    assert np.array_equal(R.numpy(), det["R"][[4, 17]])
    for i in (0, 33, 59):
        Ki, Ei, w = rank.re_ranking_encode_reference(det["D"][i], det["R"], i, 8)
        assert Ki == det["K"][i] and np.array_equal(Ei, det["E"][i])
        assert np.array_equal(w, det["V"][i, Ei])


# ------------------------------------------------------------------------------------------------------------ engine
def _tiny_log(tmp, re_ranking):
    from helpers import tiny_common, tiny_experiment, tiny_factory
    from flpr_b200.runtime.experiment import ExperimentStage
    common = tiny_common(str(tmp))
    common["defaults"]["exp_opts"].update(comm_rounds=1, val_interval=1)
    cfg = tiny_experiment(common, "fedavg")
    if re_ranking is not None:
        cfg["engine_opts"]["re_ranking"] = re_ranking
    with ExperimentStage(common, [cfg], source_factory=tiny_factory()) as stage:
        log = stage.run_experiment(cfg)
    return log.records["data"]


def test_experiment_logs_re_ranked_metrics_next_to_the_plain_ones(tmp_path):
    plain = _tiny_log(tmp_path / "off", None)
    rr = _tiny_log(tmp_path / "on", True)
    rr_keys = {"val_rr_rank_1", "val_rr_rank_3", "val_rr_rank_5", "val_rr_rank_10", "val_rr_map"}
    n_val = 0
    assert plain.keys() == rr.keys()
    for client, rounds in plain.items():
        for rnd, tasks in rounds.items():
            for task, rec in tasks.items():
                got = rr[client][rnd][task]
                assert not any(k.startswith("val_rr_") for k in rec)          # option off: no new keys
                for k, v in rec.items():
                    if k.startswith("val_"):
                        n_val += 1
                        assert got[k] == v, (client, rnd, task, k)           # bitwise: the plain path is untouched
                if "val_map" in rec:
                    assert rr_keys <= got.keys()
                    assert all(0.0 <= got[k] <= 1.0 for k in rr_keys)
    assert n_val >= 2 * 2 * 5


def test_sharded_validation_with_re_ranking_raises_on_two_ranks(tmp_path):
    script = os.path.join(os.path.dirname(__file__), "dist_rerank_check.py")
    env = dict(os.environ, FLPR_TMP=str(tmp_path), OMP_NUM_THREADS="2")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--local-addr", "127.0.0.1",
                        "--nproc-per-node", "2", script], env=env, capture_output=True, text=True, timeout=600)
    assert r.stdout.count("DIST_RERANK OK") == 2, r.stdout[-2000:] + r.stderr[-2000:]

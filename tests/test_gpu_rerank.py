"""k-reciprocal re-ranking on the H100: every stage of ``csrc/rerank.cu`` against the float64 reference on the device's
own ``D`` (so that GEMM rounding cannot flip near-tied neighbours), at N ~ 2,000, at full Market-1501 scale (distance
and top-k in full, the encoding on sampled rows), end to end at N ~ 5,000, and one experiment with the option on."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from helpers import tiny_common, tiny_experiment  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _device_distance(q, g):
    from flpr_b200.ops import rank
    x = torch.cat([q, g]).float().contiguous()
    return rank.rr_distance(rank.similarity(x, x, precise=True).contiguous(), x)


def test_stages_match_the_reference_at_n_2000():
    from flpr_b200.data.synthetic import clustered_features
    from flpr_b200.ops import rank
    q, _, g, _ = clustered_features(400, 1600, 256, 150, seed=11, device=DEV)
    n = 2000
    D = _device_distance(q, g)
    assert (D.double() - rank.re_ranking_distance_reference(q, g)).abs().max().item() < 5e-5
    R = rank.rr_topk(D, 20)
    V = rank.rr_encode(D, R, 20)
    Vq = rank.rr_expand(V, R, 6)
    out = rank.rr_jaccard(Vq, D, 400, 0.3)
    ref, det = rank.re_ranking_reference(q, g, 20, 6, 0.3, distance=D, details=True)
    assert np.array_equal(R.cpu().numpy(), det["R"])
    assert np.abs(V.dense(n).cpu().numpy() - det["V"]).max() < 1e-6
    assert np.abs(Vq.dense(n).cpu().numpy() - det["Vq"]).max() < 1e-6
    assert (out.double() - ref).abs().max().item() < 1e-5
    tiled = rank.rr_jaccard(Vq, D, 400, 0.3, tile=300)                  # six gallery tiles per query
    assert (tiled.double() - ref).abs().max().item() < 1e-5


def test_distance_topk_and_sampled_encoding_at_market1501_scale():
    from flpr_b200.data.synthetic import clustered_features
    from flpr_b200.ops import rank
    nq, ng, k1 = 3368, 15913, 20
    q, _, g, _ = clustered_features(nq, ng, 2048, 750, seed=5, device=DEV)
    D = _device_distance(q, g)
    ref_d = rank.re_ranking_distance_reference(q, g)
    assert (D.double() - ref_d).abs().max().item() < 5e-5
    del ref_d
    R = rank.rr_topk(D, k1)
    assert torch.equal(R.long(), rank.re_ranking_topk_reference(D, k1))
    V = rank.rr_encode(D, R, k1)
    Rn = R.cpu().numpy()
    rows = torch.randperm(nq + ng, generator=torch.Generator().manual_seed(0))[:256].tolist()
    cols, vals, nnz = V.cols.cpu(), V.vals.cpu(), V.nnz.cpu()
    for i in rows:
        _, E, w = rank.re_ranking_encode_reference(D[i], Rn, i, k1)
        k = int(nnz[i])
        assert np.array_equal(cols[i, :k].numpy(), E), i
        assert np.abs(vals[i, :k].double().numpy() - w).max() < 1e-6, i


def test_re_ranking_end_to_end_is_reproducible_and_ranks_like_the_reference():
    from flpr_b200.data.synthetic import clustered_features
    from flpr_b200.ops import rank
    q, ql, g, gl = clustered_features(1000, 4000, 512, 300, seed=7, device=DEV)
    a = rank.re_ranking(q, g)
    b = rank.re_ranking(q, g)
    assert a.shape == (1000, 4000) and torch.equal(a, b)
    params = {"k1": 20, "k2": 6, "lambda_value": 0.3}
    cmc, m_ap = rank.evaluate(q, ql, g, gl, re_ranking=params)
    final_ref = rank.re_ranking_reference(q, g, distance=_device_distance(q, g), **params)
    assert (a.double() - final_ref).abs().max().item() < 1e-5
    ref_cmc, ref_map = rank.rank_metrics_reference(-final_ref, ql, gl)
    assert np.abs(cmc - ref_cmc).max() <= 2e-3 and abs(m_ap - ref_map) <= 1e-3, (m_ap, ref_map)
    plain = rank.evaluate(q, ql, g, gl)
    assert m_ap > 0.5 and plain[1] > 0.5


def test_experiment_on_gpu_with_re_ranking(tmp_path):
    from flpr_b200.data.synthetic import synthetic_source_factory
    from flpr_b200.ops import native
    from flpr_b200.runtime.experiment import ExperimentStage
    common = tiny_common(str(tmp_path), device=DEV)
    common["defaults"]["task_opts"]["augment_opts"]["img_size"] = [64, 32]
    common["defaults"]["task_opts"]["loader_opts"]["batch_size"] = 8
    cfg = tiny_experiment(common, "fedavg")
    cfg["engine_opts"]["re_ranking"] = {"k1": 6, "k2": 3, "lambda_value": 0.3}
    before = native.launches()
    with ExperimentStage(common, [cfg], source_factory=synthetic_source_factory(num_ids=4, train_per_id=4,
                                                                                size=(64, 32))) as stage:
        log = stage.run_experiment(cfg)
    assert native.launches() - before > 50
    n_rr = 0
    for client in log.records["data"].values():
        for tasks in client.values():
            for vals in tasks.values():
                if "val_map" in vals:
                    n_rr += 1
                    for k in ("val_rr_rank_1", "val_rr_rank_3", "val_rr_rank_5", "val_rr_rank_10", "val_rr_map"):
                        assert 0.0 <= vals[k] <= 1.0, (k, vals[k])
    assert n_rr >= 4

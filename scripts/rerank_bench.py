"""Device time of k-reciprocal re-ranking (``ops/rank.py:re_ranking``, ``csrc/rerank.cu``) per stage and in total, at
Market-1501 scale on seeded synthetic clustered features: Q = 3,368 queries, G = 15,913 gallery images, C = 2,048
(ResNet-50 embeddings), 750 identities, noise 4.5 times the identity centre's norm (plain ranking is far from
perfect). CUDA events around every stage, after warm-up; the card's name and power limit are read in the same run. Plain and re-ranked mAP / rank-1 are reported with the times.

    python scripts/rerank_bench.py [--reps 5] [--warmup 2] [--query 3368 --gallery 15913 --dim 2048 --ids 750]

Prints one JSON line. Needs a CUDA device."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def power_limit() -> str:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--query", type=int, default=3368)
    ap.add_argument("--gallery", type=int, default=15913)
    ap.add_argument("--dim", type=int, default=2048)
    ap.add_argument("--ids", type=int, default=750)
    ap.add_argument("--spread", type=float, default=4.5)       # noise norm / centre norm
    ap.add_argument("--k1", type=int, default=20)
    ap.add_argument("--k2", type=int, default=6)
    ap.add_argument("--lambda-value", type=float, default=0.3)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rerank_bench.py measures the CUDA kernels: no CUDA device")
    from flpr_b200.data.synthetic import clustered_features
    from flpr_b200.ops import rank
    dev = torch.device("cuda", torch.cuda.current_device())
    q, ql, g, gl = clustered_features(args.query, args.gallery, args.dim, args.ids, seed=0, spread=args.spread,
                                      device=dev)
    nq = args.query
    k1, k2, lam = rank.check_re_ranking_params(args.k1, args.k2, args.lambda_value)

    stages = ["similarity", "distance", "topk", "encode", "expand", "index", "jaccard"]

    def run_once(ev):
        x = torch.cat([q, g]).float().contiguous()
        ev[0].record()
        S = rank.similarity(x, x, precise=True).contiguous()
        ev[1].record()
        D = rank.rr_distance(S, x)
        ev[2].record()
        R = rank.rr_topk(D, k1)
        ev[3].record()
        V = rank.rr_encode(D, R, k1)
        ev[4].record()
        Vq = rank.rr_expand(V, R, k2)
        ev[5].record()
        rank.rr_index(Vq, nq)                 # (timed on its own; rr_jaccard builds the index it uses again)
        ev[6].record()
        out = rank.rr_jaccard(Vq, D, nq, lam)
        ev[7].record()
        return out, V, Vq

    for _ in range(args.warmup):
        run_once([torch.cuda.Event(enable_timing=True) for _ in range(8)])
    torch.cuda.synchronize()
    times = {s: [] for s in stages}
    totals = []
    out = V = Vq = None
    for _ in range(args.reps):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(8)]
        out, V, Vq = run_once(ev)
        torch.cuda.synchronize()
        for k, s in enumerate(stages):
            t = ev[k].elapsed_time(ev[k + 1])
            if s == "jaccard":
                t -= times["index"][-1]       # rr_jaccard = index + Jaccard kernel: report the kernel alone
            times[s].append(t)
        totals.append(ev[0].elapsed_time(ev[7]) - times["index"][-1])

    # one public call, as a user runs it (the index is built once there)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    final = rank.re_ranking(q, g, k1, k2, lam)
    e1.record()
    torch.cuda.synchronize()
    assert torch.equal(final, out), "re-ranking is not reproducible from run to run"

    plain_cmc, plain_map = rank.evaluate(q, ql, g, gl)
    rr_cmc, rr_map = rank.rank_metrics(-final, ql, gl)
    med = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    res = {
        "bench": "rerank", "device": torch.cuda.get_device_name(dev), "power_limit": power_limit(),
        "Q": nq, "G": args.gallery, "C": args.dim, "ids": args.ids, "k1": k1, "k2": k2, "lambda_value": lam,
        "reps": args.reps, "stage_ms_median": {s: round(med(times[s]), 3) for s in stages},
        "total_ms_median": round(med(totals), 3), "total_ms_min": round(min(totals), 3),
        "re_ranking_call_ms": round(e0.elapsed_time(e1), 3),
        "nnz_V_mean": float(V.nnz.float().mean()), "nnz_Vq_mean": float(Vq.nnz.float().mean()),
        "peak_mem_gb": round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2),
        "plain": {"mAP": round(plain_map, 5), "rank1": round(float(plain_cmc[0]), 5)},
        "re_ranked": {"mAP": round(rr_map, 5), "rank1": round(float(rr_cmc[0]), 5)},
    }
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()

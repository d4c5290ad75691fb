"""Device time of one robust-aggregation collective (``FedComm.reduce_robust``, ``fed_reduce_robust_kernel`` in
``csrc/fedcomm.cu``) per rule, at the FedAvg ResNet-50 upload size: the upload prefix of the arena of the model in
``configs/b200/experiment_fedavg_res50_2.yaml``, read from the built model. The weighted mean the aggregators replace
(``FedComm.reduce_bcast``, ``fed_reduce_bcast_kernel``) is timed at the same K as the yardstick.

Achieved bandwidth counts the bytes each call must move per element: the K uploads read (4K B) and the result written
to every rank (4 * world B). One GPU (world 1), K in {2, 8, 32} by default. CUDA events around ``--iters``
back-to-back calls after warm-up, median of ``--reps`` windows; the card's name and power limit are read in the same
run.

    python scripts/robust_agg_bench.py [--ks 2,8,32] [--reps 5] [--iters 10] [--warmup 3]

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
    ap.add_argument("--ks", default="2,8,32")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("robust_agg_bench.py measures the CUDA kernel: no CUDA device")
    from flpr_b200.methods.fedbase import trim_count
    from flpr_b200.parallel.comm import FedComm
    from flpr_b200.runtime.builder import parser_model
    dev = torch.device("cuda", torch.cuda.current_device())
    cfg = {"name": "resnet50", "num_classes": 8000, "last_stride": 1, "neck": "bnneck",
           "fine_tuning": ["base.layer4", "classifier"]}
    model = parser_model("fedavg", cfg, dev, {"compute_dtype": "bf16"})
    n = model.arena.prefix_numel or model.arena.numel
    del model
    torch.cuda.empty_cache()

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        per_call = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            per_call.append(e0.elapsed_time(e1) / args.iters)
        return sorted(per_call)[len(per_call) // 2], min(per_call)

    results = {}
    for K in [int(k) for k in args.ks.split(",")]:
        comm = FedComm(dev, K, arena_bytes=(K + 1) * n * 4 + (64 << 20))
        comm.alloc_client_buffer("up", n)
        comm.alloc_client_buffer("cnt", 4)
        comm.alloc_rank_buffer("glob", n)
        g = torch.Generator(device=dev).manual_seed(K)
        for c in range(K):
            comm.client_view("up", c).normal_(generator=g)
            comm.client_view("cnt", c).fill_(float(100 + c))
        clients = list(range(K))
        nbytes = (4 * K + 4 * comm.world) * n
        row = {}
        cases = {"median": lambda: comm.reduce_robust("up", "glob", clients, "median"),
                 "trimmed_mean_0.1": lambda: comm.reduce_robust("up", "glob", clients, "trimmed_mean",
                                                                trim_count(0.1, K)),
                 "reduce_bcast": lambda: comm.reduce_bcast("up", "glob", clients, cnt="cnt")}
        for name, fn in cases.items():
            med, best = timed(fn)
            row[name] = {"ms_median": round(med, 4), "ms_min": round(best, 4),
                         "GB_per_s_median": round(nbytes / (med * 1e-3) / 1e9, 1)}
        comm.check_errors()
        results[str(K)] = dict(row, bytes=nbytes)
        comm.close()
        del comm
        torch.cuda.empty_cache()
    res = {"bench": "robust_agg", "device": torch.cuda.get_device_name(dev), "power_limit": power_limit(),
           "world": 1, "numel": n, "MB_fp32": round(n * 4 / 1e6, 1), "reps": args.reps, "iters": args.iters,
           "K": results}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()

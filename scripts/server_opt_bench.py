"""Device time of one server-optimizer step (``ops/fused.py:server_opt_step``, ``server_opt_kernel`` in
``csrc/fused_ops.cu``) per rule, at the FedAvg ResNet-50 upload size: the upload prefix of the arena of the model in
``configs/b200/experiment_fedavg_res50_2.yaml``, read from the built model. Also times what the step replaces without
``server_opt`` (copy of the mean into the replica + bf16 refresh of the replica's arena).

Achieved bandwidth counts the bytes the rule must move per element: ``sgd`` reads x, mean, m (12 B) and writes x, m
(8 B); ``adagrad`` / ``adam`` / ``yogi`` also read and write v (16 B read, 12 B written); every rule writes the bf16 copy
of x (2 B). CUDA events around ``--iters`` back-to-back steps after warm-up, median of ``--reps`` windows; the card's
name and power limit are read in the same run.

    python scripts/server_opt_bench.py [--reps 5] [--iters 20] [--warmup 5]

Prints one JSON line. Needs a CUDA device."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

BYTES_PER_ELEMENT = {"sgd": 12 + 8 + 2, "adagrad": 16 + 12 + 2, "adam": 16 + 12 + 2, "yogi": 16 + 12 + 2}


def power_limit() -> str:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("server_opt_bench.py measures the CUDA kernel: no CUDA device")
    from flpr_b200.ops import fused as fops
    from flpr_b200.runtime.builder import parser_model
    dev = torch.device("cuda", torch.cuda.current_device())
    cfg = {"name": "resnet50", "num_classes": 8000, "last_stride": 1, "neck": "bnneck",
           "fine_tuning": ["base.layer4", "classifier"]}
    arena = parser_model("fedavg", cfg, dev, {"compute_dtype": "bf16"}).arena
    n = arena.prefix_numel or arena.numel
    g = torch.Generator(device=dev).manual_seed(0)
    x = arena.master[:n]
    mean = (x + 1e-3 * torch.randn(n, device=dev, generator=g)).contiguous()
    m, v = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    shadow = arena.shadow[:n]
    hp = {"lr": 1e-3, "momentum": 0.9, "beta1": 0.9, "beta2": 0.99, "tau": 1e-3}

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        per_step = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            per_step.append(e0.elapsed_time(e1) / args.iters)
        return sorted(per_step)[len(per_step) // 2], min(per_step)

    rules = {}
    for rule in ("sgd", "adagrad", "adam", "yogi"):
        med, best = timed(lambda: fops.server_opt_step(rule, x, mean, m, None if rule == "sgd" else v, x_bf16=shadow,
                                                       **hp))
        rules[rule] = {"ms_median": round(med, 4), "ms_min": round(best, 4),
                       "bytes": BYTES_PER_ELEMENT[rule] * n,
                       "GB_per_s_median": round(BYTES_PER_ELEMENT[rule] * n / (med * 1e-3) / 1e9, 1)}

    def plain():
        arena.master[:n].copy_(mean)
        arena.refresh_shadow()
    med, best = timed(plain)
    res = {"bench": "server_opt", "device": torch.cuda.get_device_name(dev), "power_limit": power_limit(),
           "numel": n, "MB_fp32": round(n * 4 / 1e6, 1), "reps": args.reps, "iters": args.iters, "rules": rules,
           "plain_copy_and_refresh": {"ms_median": round(med, 4), "ms_min": round(best, 4),
                                      "refresh_numel": arena.numel}}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()

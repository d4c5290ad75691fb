"""Device cost of Synaptic Intelligence (``methods/si.py``) on the ResNet-50 trainable arena (``fine_tuning`` =
``base.layer4`` + ``classifier``, as in ``configs/b200/experiment_si_res50_1.yaml``; the size is read from a built
``si`` model):

* the penalised Adam step (``fused_opt_kernel``) without and with the path integral ``omega``, alternated window by
  window in one process;
* one consolidation at a task switch (``Model.switch_task``: fp32 tensor ops);
* for comparison, what EWC does instead after every task: one ``remember_task`` Fisher pass (forward / backward per
  batch) over ``--images`` synthetic images.

Achieved bandwidth counts the bytes each step variant must move per element: the penalised Adam step reads p, g, m, v,
Q, R (24 B), writes p, m, v (12 B) and the bf16 copy of p (2 B): 38 B; the path integral reads and writes W: 8 B more.
CUDA events around ``--iters`` back-to-back steps after warm-up, median of ``--reps`` windows; the card's name and power
limit are read in the same run.

    python scripts/si_bench.py [--reps 7] [--iters 20] [--warmup 5] [--images 512]

Prints one JSON line. Needs a CUDA device."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

BYTES_PENALISED_ADAM = 24 + 12 + 2
BYTES_SI = 8


def power_limit() -> str:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def window_ms(fn, iters: int) -> float:
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--images", type=int, default=512, help="images of the task EWC's Fisher pass runs over")
    ap.add_argument("--batch", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("si_bench.py measures CUDA kernels: no CUDA device")
    from flpr_b200.methods import ewc
    from flpr_b200.runtime.arena import ArenaOptimizer
    from flpr_b200.runtime.builder import parser_criterion, parser_model
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(0)
    cfg = {"name": "resnet50", "num_classes": 8000, "last_stride": 1, "neck": "bnneck", "lambda_penalty": 0.1,
           "si_xi": 1e-3, "fine_tuning": ["base.layer4", "classifier"]}
    model = parser_model("si", cfg, dev, {"compute_dtype": "bf16"})
    a = model.arena
    n = a.numel
    opt = ArenaOptimizer("adam", a, lr=1e-3, weight_decay=1e-5)
    model.switch_task("task-0")
    a.grad.normal_(0.0, 1e-3)
    model.F.uniform_(0.0, 1.0)                         # a penalty that is active (non-zero Q / R)
    model.rebuild_penalty()
    model.install(opt)
    W = model.W

    def step_plain():
        opt.omega = None
        opt.step()

    def step_si():
        opt.omega = W
        opt.step()

    for _ in range(args.warmup):
        step_plain()
        step_si()
    torch.cuda.synchronize()
    plain, si = [], []
    for _ in range(args.reps):                          # alternated: both see the same clocks and neighbours
        plain.append(window_ms(step_plain, args.iters))
        si.append(window_ms(step_si, args.iters))
    med = lambda xs: sorted(xs)[len(xs) // 2]  # noqa: E731

    def consolidate():                                  # every call is a task switch
        model.switch_task("b" if model.task_name == "a" else "a")
    for _ in range(args.warmup):
        consolidate()
    torch.cuda.synchronize()
    cons = [window_ms(consolidate, 5) for _ in range(args.reps)]

    # EWC: Fisher pass over one remembered task (the current task is skipped, so a second task triggers it)
    em = parser_model("ewc", dict(cfg, lambda_penalty=50.0), dev, {"compute_dtype": "bf16"})
    crit = parser_criterion({"name": "cross_entropy", "num_classes": 8000, "epsilon": 0.1})
    em.operator = ewc.Operator(criterion=crit, optimizer=ArenaOptimizer("adam", em.arena, lr=1e-3))
    g = torch.Generator(device=dev).manual_seed(1)
    batches = [(torch.randn(args.batch, 3, 256, 128, device=dev, generator=g),
                torch.randint(0, 8000, (args.batch,), device=dev, generator=g), None)
               for _ in range(args.images // args.batch)]
    em.train()
    em.remember_task("task-0", batches)                 # skipped task: nothing computed
    em.remember_task("task-1", batches)                 # warm-up: one pass over task-0
    torch.cuda.synchronize()
    fisher = []
    for _ in range(3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record()
        em.calculate()                                  # what remember_task runs: one pass over task-0's images
        e1.record()
        torch.cuda.synchronize()
        fisher.append((e0.elapsed_time(e1), (time.perf_counter() - t0) * 1e3))
    fisher.sort()

    mp, ms = med(plain), med(si)
    out = {
        "gpu": torch.cuda.get_device_name(dev), "power_limit": power_limit(), "arena_elements": n,
        "adam_penalty_step": {"ms_median": round(mp, 4), "ms_min": round(min(plain), 4),
                              "bytes": BYTES_PENALISED_ADAM * n,
                              "GB_per_s_median": round(BYTES_PENALISED_ADAM * n / (mp * 1e-3) / 1e9, 1)},
        "adam_penalty_si_step": {"ms_median": round(ms, 4), "ms_min": round(min(si), 4),
                                 "bytes": (BYTES_PENALISED_ADAM + BYTES_SI) * n,
                                 "GB_per_s_median": round((BYTES_PENALISED_ADAM + BYTES_SI) * n / (ms * 1e-3) / 1e9, 1)},
        "si_step_overhead_ms_median": round(ms - mp, 4),
        "consolidation_ms_median": round(med(cons), 4),
        "ewc_fisher_pass": {"images": len(batches) * args.batch, "ms_median": round(fisher[1][0], 2),
                            "host_ms_median": round(fisher[1][1], 2)},
        "reps": args.reps, "iters": args.iters,
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()

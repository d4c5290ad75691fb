"""Headline benchmark: FedSTIL, ResNet-50, 8 clients, 256x128 crops, one *step* = one federated communication round.

    python bench.py --gpus N --steps K --warmup W [--impl flpr|reference|nccl]

A round (``experiment.py:183-243`` of the reference) = similarity-weighted dispatch to every client -> local training
of every client (frozen-trunk prototype pass + head training incl. prototype rehearsal + herding) -> theta uploads ->
FedAvg aggregation into the server model, with the reference's checkpoint files written every round.
``value`` = images/s summed over all clients (whole job), device-timed with CUDA events, max over ranks.
``e2e``   = the same metric measured by wall clock around the public API (``ExperimentStage`` rounds): every batch is
copied host->device from pinned memory and every epoch's loss/accuracy is read back.

``--impl reference`` runs the UNMODIFIED reference installed in ``oracle/_ref`` through its own builder /
``ExperimentStage._process_one_round`` on the same synthetic workload. ``--impl nccl`` runs this engine with the
collectives expressed as plain ``torch.distributed`` (NCCL) calls – the "baseline, not the product" harness.
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "images/sec aggregate over 8 clients (FedSTIL ResNet-50 federated round, 256x128)"

# method-specific ``model_opts`` (the values of configs/b200/*.yaml) and the checkpoint name of the reference's configs
METHOD_MODEL_OPTS = {
    "fedstil": {"atten_default": 0.9, "lambda_l1": 1e-3},
    "fedstil-atten": {"atten_default": 0.9, "lambda_l1": 1e-3},
    "fedweit": {"lambda_l1": 1e-3, "lambda_l2": 100.0, "lambda_mask": 0.0, "kb_cnt": 5},
    "fedprox": {"lambda_l2": 1e-2},
    "fedcurv": {"lambda_penalty": 10.0},
    "ewc": {"lambda_penalty": 50.0},
    "mas": {"lambda_penalty": 0.01},
    "icarl": {"n_classes": 10},
}
LOCAL_ONLY = ("baseline", "ewc", "mas", "icarl")          # single-client lifelong methods (BASELINE config 5)


def metric_name(a) -> str:
    if a.method == "fedstil" and a.model == "resnet50" and a.clients == 8:
        return METRIC
    return (f"images/sec aggregate over {a.clients} clients ({a.method} {a.model} federated round, "
            f"{a.height}x{a.width})")


def _layer_kernel_status():
    """Which ``csrc/layer_ops.cu`` families (weight composition, Swin token kernels, dispatch apply) were consulted by
    this run and whether they passed their on-device self-check (empty: the method / model uses none of them)."""
    try:
        from flpr_b200.ops import layer as lops
        return lops.status()
    except Exception:  # noqa: BLE001
        return {}


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="flpr", choices=["flpr", "reference", "nccl"])
    ap.add_argument("--clients", type=int, default=8)
    ap.add_argument("--images", type=int, default=512, help="train images per client task")
    ap.add_argument("--ids", type=int, default=64, help="identities per client task")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--epochs", type=int, default=1)
    ap.add_argument("--model", default="resnet50")
    ap.add_argument("--method", default="fedstil",
                    help="federated / continual method (BASELINE configs 3 and 5: fedcurv, ewc, mas, icarl, ...)")
    ap.add_argument("--height", type=int, default=256)
    ap.add_argument("--width", type=int, default=128)
    ap.add_argument("--parallel", type=int, default=3,
                    help="clients trained concurrently per device (common.yaml `parallel`; the reference arm keeps its "
                         "shipped default of 1)")
    ap.add_argument("--no-ckpt", action="store_true", help="disable checkpoint files (not the headline config)")
    ap.add_argument("--payload-ring", type=int, default=2,
                    help="rounds of per-round payload checkpoints kept on the RAM disk (older rounds are recycled in "
                         "place; the harness used to unlink them - a long run must not fill the RAM disk)")
    ap.add_argument("--staged-ckpt", action="store_true", help="round-1 checkpoint pipeline (pinned arena + writer "
                                                               "processes) instead of DMA into mapped files")
    ap.add_argument("--dtype", default="bf16", choices=["bf16", "fp32"],
                    help="compute dtype of the engine: bf16 = the product path (tensor-core kernels, fp32 masters); fp32 = "
                         "the same engine with fp32 activations / weights on the library kernels (the precision-matched "
                         "arm for convergence comparisons with the fp32 reference; not the headline)")
    ap.add_argument("--cpu-debug", action="store_true", help="tiny CPU run to exercise the harness")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed rounds, write what the last timed round computed (server and client "
                         "parameters, per-client training loss / accuracy) as DIR/<name>.npy")
    return ap.parse_args()


class ClockSampler:
    """nvidia-smi clocks / throttle reasons DURING the timed region."""

    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index: int):
        self.idx = gpu_index
        self.proc = None
        self.lines = []

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "200", "-i", str(self.idx)], stdout=subprocess.PIPE, text=True)
            threading.Thread(target=self._pump, daemon=True).start()
        except Exception:
            self.proc = None

    def _pump(self):
        for ln in self.proc.stdout:
            self.lines.append(ln.strip())

    def stop(self) -> dict:
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        sm, mx, reasons = [], 0, set()
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1]))
                mx = max(mx, float(f[2]))
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": mx or None, "reasons": sorted(reasons),
                "samples": len(sm)}


def ckpt_root() -> str:
    base = "/dev/shm" if os.path.isdir("/dev/shm") else "/tmp"
    return os.path.join(base, f"flpr_bench_{os.getpid()}")


def build_config(a, impl: str, world: int):
    """Common + experiment config (same numbers for both arms)."""
    root = ckpt_root()
    common = {"datasets_dir": os.path.join(root, "data"), "checkpoints_dir": os.path.join(root, "ckpts"),
              "logs_dir": os.path.join(root, "logs"), "parallel": 1 if impl == "reference" else max(1, a.parallel),
              "device": ["cpu"] if a.cpu_debug else [f"cuda:{i}" for i in range(max(a.gpus, 1))],
              "defaults": {}}
    exp = {
        "exp_name": f"bench-{a.method}", "exp_method": a.method, "random_seed": 123,
        "exp_opts": {"comm_rounds": 10 ** 6, "val_interval": 10 ** 9, "online_clients": a.clients},
        "model_opts": {"name": a.model, "num_classes": 8000, "neck": "bnneck",
                       **({} if a.model.startswith("swin") else {"last_stride": 1}),
                       **METHOD_MODEL_OPTS.get(a.method, {}),
                       **({"lambda_k": a.images} if a.method.startswith("fedstil") else {}),
                       **({"k": a.images} if a.method == "icarl" else {}),
                       "fine_tuning": ["base.layers.3", "classifier"] if a.model.startswith("swin")
                       else ["base.layer4", "classifier"]},
        "criterion_opts": {"name": "cross_entropy", "num_classes": 8000, "epsilon": 0.1},
        "optimizer_opts": {"name": "adam", "lr": 1e-3, "weight_decay": 1e-5},
        "scheduler_opts": {"name": "step_lr", "step_size": 5},
        "task_opts": {"sustain_rounds": 10 ** 6, "train_epochs": a.epochs,
                      "augment_opts": {"level": "default", "img_size": [a.height, a.width],
                                       "norm_mean": [0.485, 0.456, 0.406], "norm_std": [0.229, 0.224, 0.225]},
                      "loader_opts": {"batch_size": a.batch, "num_workers": 0, "pin_memory": False,
                                      "persistent_workers": False, "multiprocessing_context": None}},
        "server": {"server_name": "server", "distance_calculate_step": 10, "distance_calculate_decay": 0.8},
        "clients": [{"client_name": f"client-{i}",
                     **({"model_ckpt_name": "fedstil_model"} if a.method.startswith("fedstil") else {}),
                     "tasks": [f"task-{i}-{t}" for t in range(5)]} for i in range(a.clients)],
        "engine_opts": {"compute_dtype": getattr(a, "dtype", "bf16"), "comm_mode": "nccl" if impl == "nccl" else None,
                        "val_at_round0": False, "checkpoints": not a.no_ckpt, "save_payload_ckpts": not a.no_ckpt,
                        "mapped_checkpoints": not a.staged_ckpt, "payload_ring": a.payload_ring},
    }
    return common, exp


def bench_config(a, impl: str, parallelism: str) -> dict:
    """The ``config`` block of the JSON line: the SAME keys and values for every arm (arm-specific remarks go to
    ``notes``), so that a config diff between the arms shows real differences only."""
    return {"model": a.model, "method": a.method, "clients": a.clients, "global_batch": a.batch * a.clients,
            "batch_per_client": a.batch, "images_per_client_task": a.images, "ids_per_task": a.ids, "seq_len": None,
            "img_size": [a.height, a.width], "epochs_per_round": a.epochs,
            "rehearsal_lambda_k": a.images if a.method.startswith("fedstil") or a.method == "icarl" else None,
            "optimizer": "adam lr 1e-3 wd 1e-5", "method_opts": METHOD_MODEL_OPTS.get(a.method, {}),
            "num_classes": 8000,
            "checkpoints": "off" if a.no_ckpt else "reference layout, every round, flushed inside the e2e region",
            "step_definition": ("one federated round: dispatch (spatial-temporal mix) + local train of all clients "
                                "(prototype pass, head training with rehearsal, herding) + upload + aggregate")
            if a.method.startswith("fedstil") else
            "one communication round of the reference's loop (experiment.py:183-243): dispatch + local train of all "
            "online clients (full backbone in train mode) + upload + aggregate",
            "l2": "inputs larger than L2 (per-round working set >> 50 MB: 8 x 400 MB client state + images)"}


def convergence_block(records: dict, rounds: int) -> dict:
    """Per-round training metrics averaged over the clients, from the experiment log both arms keep
    (``data.{client}.{round}.{task}.{tr_acc,tr_loss}``): the evidence that the two arms train the same model."""
    data = (records or {}).get("data", {})
    acc, loss = [], []
    for r in range(1, rounds + 1):
        a_, l_ = [], []
        for per_round in data.values():
            for task in (per_round.get(r) or per_round.get(str(r)) or {}).values():
                if "tr_acc" in task:
                    a_.append(float(task["tr_acc"]))
                    l_.append(float(task["tr_loss"]))
        if a_:
            acc.append(round(100.0 * sum(a_) / len(a_), 2))
            loss.append(round(sum(l_) / len(l_), 4))
    return {"rounds": len(acc), "tr_acc_pct": acc, "tr_loss": loss,
            "final_tr_acc_pct": acc[-1] if acc else None, "final_tr_loss": loss[-1] if loss else None}


DUMP_SAMPLE = 1 << 20          # elements kept per parameter arena by --dump-outputs (4 MB each in float32)


def dump_outputs(out_dir: str, server, clients, records: dict, rnd: int) -> None:
    """What a round hands its caller: the aggregated server parameters, every client's parameters and the per-client
    training loss / accuracy of round ``rnd``. An arena larger than ``DUMP_SAMPLE`` elements is reduced to a fixed,
    seeded sample of its elements (the same indices for the same arena size), so the files stay within 64 MB."""
    import numpy as np
    import torch
    os.makedirs(out_dir, exist_ok=True)

    def arena(name, model):
        flat = model.arena.master.detach().reshape(-1)
        if flat.numel() > DUMP_SAMPLE:
            g = torch.Generator().manual_seed(0)
            idx = torch.randint(0, flat.numel(), (DUMP_SAMPLE,), generator=g).to(flat.device)
            flat = flat[idx]
        np.save(os.path.join(out_dir, f"{name}.npy"), flat.float().cpu().numpy())

    arena("server_params", server.model)
    loss, acc = [], []
    for i, c in enumerate(clients):
        arena(f"client{i}_params", c.model)
        per_round = (records.get("data", {}).get(c.client_name) or {})
        tasks = per_round.get(rnd) or per_round.get(str(rnd)) or {}
        loss.append([float(t["tr_loss"]) for t in tasks.values() if "tr_loss" in t])
        acc.append([float(t["tr_acc"]) for t in tasks.values() if "tr_acc" in t])
    np.save(os.path.join(out_dir, "train_loss.npy"), np.asarray(loss, dtype=np.float64))
    np.save(os.path.join(out_dir, "train_acc.npy"), np.asarray(acc, dtype=np.float64))


def cleanup_payloads(ckpt_dir: str) -> None:
    """Per-round payload files are unique per round; drop them between steps (outside the timed region) so that a
    long run cannot fill the RAM disk. Model checkpoints (overwritten in place) stay."""
    for d, _, files in os.walk(ckpt_dir):
        for f in files:
            if f[:1].isdigit() and f.endswith(".ckpt"):
                try:
                    os.remove(os.path.join(d, f))
                except OSError:
                    pass


# ================================================================================================== flpr / nccl arms
def run_flpr(a, impl: str) -> dict:
    import torch
    import torch.distributed as dist
    from flpr_b200.data.synthetic import random_array_split
    from flpr_b200.ops import native
    from flpr_b200.runtime.config import merge_experiment
    from flpr_b200.runtime.experiment import ExperimentStage
    from flpr_b200.runtime.explog import ExperimentLog
    from flpr_b200.utils.misc import DeviceTimer, same_seeds
    from flpr_b200.utils.trace import d2h_bytes

    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    common, exp = build_config(a, impl, world)
    cfg = merge_experiment(common, exp)
    size = (a.height, a.width)

    def factory(task: str, split: str):
        cid = int(task.split("-")[1])
        tid = int(task.split("-")[2])
        n = a.images if split == "train" else 64
        return random_array_split(n, a.ids, size, id_offset=(cid * 5 + tid) * a.ids % (8000 - a.ids),
                                  seed=cid * 100 + tid * 3 + {"train": 0, "query": 1, "gallery": 2}[split])

    with ExperimentStage(common, [cfg], source_factory=factory) as stage:
        same_seeds(cfg["random_seed"])
        dev = stage.device
        store, comm, server, clients, names = stage.build(cfg)
        log = ExperimentLog(os.path.join(common["logs_dir"], "bench.json"), enabled=False)
        timer = DeviceTimer(dev)
        cuda = dev.type == "cuda"

        def sync():
            if cuda:
                torch.cuda.synchronize(dev)
            if world > 1:
                dist.barrier()

        # Harness housekeeping, NOT part of a federated round: per-round payload files have unique names, so a long
        # run would fill the RAM disk. A background thread unlinks the payload files of finished rounds.
        import queue as _q
        janitor_q: "_q.Queue" = _q.Queue()

        def janitor():
            while janitor_q.get() is not None:
                cleanup_payloads(common["checkpoints_dir"])

        jt = threading.Thread(target=janitor, daemon=True)
        jt.start()

        ringed = getattr(store, "mapped", False) and getattr(store, "payload_ring", 0) > 0

        def one_round(r):
            stage._process_one_round(r, server, clients, names, cfg, log, timer, comm)
            if rank == 0 and r % 2 == 0 and not ringed:
                janitor_q.put(r)

        def after_round():
            store.flush()
            if rank == 0 and not ringed:
                cleanup_payloads(common["checkpoints_dir"])

        r = 0
        for _ in range(a.warmup):
            r += 1
            one_round(r)
            sync()
            after_round()
        sampler = ClockSampler(dev.index or 0) if cuda and rank == 0 else None

        # ---- device-timed region: exactly K rounds ---------------------------------------------------------------
        sync()
        if sampler:
            sampler.start()
        launches0 = native.launches()
        h2d0 = sum(getattr(t["tr_loader"], "h2d_bytes", 0) for c in clients for t in c.task_pipeline._cache.values())
        if cuda:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        t0 = time.perf_counter()
        for _ in range(a.steps):
            r += 1
            one_round(r)
        store.flush()               # every checkpoint byte of the timed rounds has left the device before the clock
        if cuda:                    # stops: a short run cannot hide snapshot traffic in a staging buffer
            e1.record()
        sync()
        wall_ms = (time.perf_counter() - t0) * 1e3
        dev_ms = e0.elapsed_time(e1) if cuda else wall_ms
        launches = native.launches() - launches0
        h2d1 = sum(getattr(t["tr_loader"], "h2d_bytes", 0) for c in clients for t in c.task_pipeline._cache.values())
        clocks = sampler.stop() if sampler else None
        if a.dump_outputs and rank == 0:
            dump_outputs(a.dump_outputs, server, clients, log.records, r)
        after_round()

        # ---- end-to-end region: K more rounds by wall clock through the public API ---------------------------------
        sync()
        ckpt0 = store.bytes_written
        d2h0 = d2h_bytes()
        t0 = time.perf_counter()
        for _ in range(a.steps):
            r += 1
            one_round(r)
        store.flush()                           # every checkpoint of these rounds is on disk before the clock stops
        sync()
        e2e_ms = (time.perf_counter() - t0) * 1e3
        d2h = float(d2h_bytes() - d2h0)         # bytes of the device tensors the rounds read back (losses, hit counts,
                                                # herding group sizes, the logged mixing matrix): counted where copied
        ckpt_bytes = float(store.bytes_written - ckpt0)          # snapshot bytes that reached the writers (flushed)
        after_round()

        red = torch.tensor([dev_ms, e2e_ms, float(launches), float(h2d1 - h2d0), ckpt_bytes, d2h], dtype=torch.float64,
                           device=dev if cuda else "cpu")
        if world > 1:
            mx = red.clone()
            dist.all_reduce(mx, op=dist.ReduceOp.MAX)
            sm = red.clone()
            dist.all_reduce(sm, op=dist.ReduceOp.SUM)
            dev_ms, e2e_ms = mx[0].item(), mx[1].item()
            launches, h2d, ckpt_bytes, d2h = int(sm[2].item()), sm[3].item(), sm[4].item(), sm[5].item()
        else:
            h2d = float(h2d1 - h2d0)
        phases = {k: round(sum(v[-2 * a.steps:]) / max(len(v[-2 * a.steps:]), 1), 3) for k, v in timer.flush().items()}
        records = log.records
        if world > 1:                                   # C7: every rank logs its own clients
            parts = [None] * world if rank == 0 else None
            dist.gather_object(log.records.get("data", {}), parts, dst=0)
            if rank == 0:
                merged = {}
                for part in parts:
                    merged.update(part or {})
                records = {"data": merged}
        conv = convergence_block(records, r)
        comm_bytes = comm.bytes_moved if comm is not None else 0
        store.close()
        janitor_q.put(None)
        jt.join(timeout=60)
        if comm is not None:
            comm.check_errors()
            comm.close()
    imgs_per_round = a.clients * a.images * a.epochs
    ms_per_step = dev_ms / a.steps
    value = imgs_per_round / (ms_per_step / 1e3)
    e2e_value = imgs_per_round / (e2e_ms / a.steps / 1e3)
    out = {
        "metric": metric_name(a), "value": round(value, 2), "unit": "images/s", "n_gpus": a.gpus, "steps": a.steps,
        "warmup": a.warmup, "ms_per_step": round(ms_per_step, 3), "higher_is_better": True, "scaling": "strong",
        "vs_baseline": None, "dtype": a.dtype if not a.cpu_debug else "fp32",
        "data": "synthetic 256x128 uint8 crops in pinned host memory, random-init weights",
        "impl": impl,
        "config": bench_config(a, impl, ""),
        "notes": {"parallelism": f"client-per-rank x{a.gpus} (8 clients round-robin, {a.parallel} concurrent client "
                                 f"streams per GPU)",
                  "semantics": "reference_compat (trained L1 anchors, per-epoch lr reset, exemplar relabelling)",
                  "timing": "CUDA events on the launching stream, max over ranks",
                  "layer_kernels": _layer_kernel_status()},
        "convergence": conv,
        "e2e": {"value": round(e2e_value, 2), "unit": "images/s", "ms_per_step": round(e2e_ms / a.steps, 3),
                "h2d_bytes_per_step": int(h2d / a.steps),
                "d2h_bytes_per_step": int(d2h / a.steps),
                "checkpoint_bytes_per_step": int(ckpt_bytes / a.steps)},
        "gpu_launches": int(launches),
        "clocks": clocks,
        "phase_ms_avg": phases,
        "comm_bytes_rank0": int(comm_bytes),
    }
    return out if rank == 0 else {}


# ================================================================================================== reference arm
def run_reference(a) -> dict:
    from baseline.reference_arm import run_reference_arm
    return run_reference_arm(a, build_config, cleanup_payloads, metric_name(a), ClockSampler, bench_config,
                             convergence_block)


def main():
    a = parse_args()
    if a.method in LOCAL_ONLY and "--clients" not in sys.argv:
        a.clients = 1
    if a.cpu_debug:
        a.model, a.images, a.ids, a.batch, a.height, a.width = "resnet18", 16, 4, 8, 64, 32
        a.clients = min(a.clients, 2)
    try:
        if a.impl == "reference":
            out = run_reference(a)
        else:
            out = run_flpr(a, a.impl)
    finally:
        shutil.rmtree(ckpt_root(), ignore_errors=True)
    if out:
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

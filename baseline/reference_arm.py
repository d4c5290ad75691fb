"""Reference arm of ``bench.py``: the UNMODIFIED reference (installed in ``oracle/_ref`` from a copy of
``/root/reference`` plus a packaging shim) driven through its own public API – ``builder.parser_server`` /
``builder.parser_clients`` / ``experiment.ExperimentStage._process_one_round`` – on the same synthetic workload.

Nothing from ``flpr_b200`` runs on this path. The only accommodations are the ones SURVEY §8 lists as required to
run the reference on a current, offline stack:
  1. ``load_state_dict_from_url`` is stubbed (no network) with a random-init torchvision ``state_dict``;
  2. ``TORCH_FORCE_NO_WEIGHTS_ONLY_LOAD=1`` (its exemplar checkpoints hold numpy objects);
  3. ``multiprocessing_context: null`` in ``loader_opts``;
and, because no dataset exists offline, every client's ``task_pipeline`` is an in-memory equivalent that hands the
reference its own ``ReIDImageDataset(source=dict)`` / ``DataLoader`` objects holding pre-normalised float tensors
(this *removes* JPEG decoding, ToTensor / Normalize / Resize from the reference's timed region – it favours the
reference; the random part of its train transform, RandomHorizontalFlip + RandomErasing, is still applied per sample
by its own torchvision transform objects, so that both arms train on augmented crops and their accuracies compare).
Multi-GPU follows the reference's own mechanism: one process, ``device: [cuda:0..N-1]``, thread pool.
"""
from __future__ import annotations

import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
_T_IMPORT = time.perf_counter()          # ~process start: bench.py imports this module first thing in the arm
REF = os.path.join(os.path.dirname(HERE), "oracle", "_ref")


def _unavailable(why: str) -> dict:
    return {"impl": "reference", "unavailable": why}


class _MemoryPipeline:
    """Duck-typed ``ReIDTaskPipeline`` (``datasets/datasets_pipeline.py``) over in-memory splits."""

    def __init__(self, task_list, task_opts, make_split, DataLoader, ReIDImageDataset):
        self.task_list = task_list
        self.task_opts = task_opts
        self.current_task_idx = -1
        self.task_round_rest = [task_opts["sustain_rounds"] for _ in task_list]
        self._make_split, self._DL, self._DS = make_split, DataLoader, ReIDImageDataset
        self._cache = {}

    def reach_final_task(self):
        return self.current_task_idx + 1 == len(self.task_list)

    def _loader(self, task, split, shuffle):
        ds = self._DS(source=self._make_split(task, split))
        if split == "train" and getattr(self, "train_transform", None) is not None:
            ds.flpr_transform = self.train_transform
        bs = self.task_opts["loader_opts"]["batch_size"]
        return self._DL(dataset=ds, shuffle=shuffle, drop_last=len(ds) % bs == 1, batch_size=bs, num_workers=0)

    def get_task(self, idx=-1):
        if idx not in self._cache:
            task = self.task_list[idx]
            self._cache[idx] = {"task_name": task, "tr_epochs": self.task_opts["train_epochs"],
                                "tr_loader": self._loader(task, "train", True),
                                "query_loader": self._loader(task, "query", False),
                                "gallery_loaders": self._loader(task, "gallery", False)}
        return self._cache[idx]

    def current_task(self):
        if self.current_task_idx == -1:
            self.current_task_idx = 0
        return self.get_task(self.current_task_idx)

    def next_task(self):
        if not self.reach_final_task():
            if self.current_task_idx != -1 and self.task_round_rest[self.current_task_idx]:
                self.task_round_rest[self.current_task_idx] -= 1
            else:
                self.current_task_idx += 1
                self.task_round_rest[self.current_task_idx] -= 1
        return self.current_task()


def run_reference_arm(a, build_config, cleanup_payloads, metric, ClockSampler, bench_config=None,
                      convergence_block=None) -> dict:
    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    if not os.path.isdir(os.path.join(REF, "methods")):
        return _unavailable("oracle/_ref is missing (the reference oracle was not built: oracle/install_reference.sh)")
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("gloo")
        if rank != 0:                       # the reference is single-process multi-device: rank 0 drives all GPUs
            dist.barrier()
            dist.destroy_process_group()
            return {}
    os.environ.setdefault("TORCH_FORCE_NO_WEIGHTS_ONLY_LOAD", "1")
    sys.path.insert(0, REF)
    for mod in [m for m in sys.modules if m.split(".")[0] in ("datasets", "models", "methods", "modules", "tools",
                                                             "criterions", "builder", "experiment")]:
        del sys.modules[mod]
    try:
        import torch
        import torchvision
        import models.resnet as ref_resnet
        import models.swin_transformer as ref_swin

        def _fake_url_loader(url, *args, **kwargs):
            name = [k for k, v in ref_resnet.model_urls.items() if v == url]
            if name:
                return getattr(torchvision.models, name[0])(weights=None).state_dict()
            raise RuntimeError("no network: unknown url " + str(url))

        ref_resnet.load_state_dict_from_url = _fake_url_loader
        ref_swin.load_state_dict_from_url = _fake_url_loader
        from builder import parser_clients, parser_server
        from datasets.datasets_loader import ReIDImageDataset
        from experiment import ExperimentLog, ExperimentStage
        from tools.utils import same_seeds
        from torch.utils.data import DataLoader
    except Exception as ex:  # pragma: no cover
        return _unavailable(f"reference import failed: {type(ex).__name__}: {ex}")

    ngpu = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if not a.cpu_debug and ngpu < a.gpus:
        return _unavailable(f"needs {a.gpus} CUDA devices, found {ngpu}")
    common, exp = build_config(a, "reference", 1)
    exp.pop("engine_opts", None)
    exp["task_opts"]["loader_opts"]["multiprocessing_context"] = None
    os.makedirs(common["checkpoints_dir"], exist_ok=True)
    os.makedirs(common["logs_dir"], exist_ok=True)
    same_seeds(exp["random_seed"])

    mean = torch.tensor([0.485, 0.456, 0.406]).view(3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225]).view(3, 1, 1)

    def make_split(task, split):
        cid, tid = int(task.split("-")[1]), int(task.split("-")[2])
        n = a.images if split == "train" else 64
        # the very bytes and labels flpr_b200.data.synthetic.random_array_split hands to the other arm (NHWC there)
        g = torch.Generator().manual_seed(cid * 100 + tid * 3 + {"train": 0, "query": 1, "gallery": 2}[split])
        imgs = torch.randint(0, 256, (n, a.height, a.width, 3), dtype=torch.uint8, generator=g).permute(0, 3, 1, 2)
        off = (cid * 5 + tid) * a.ids % (8000 - a.ids)
        pids = (torch.randint(0, a.ids, (n,), generator=g) + off).tolist()
        src = {}
        for i, pid in enumerate(pids):
            src.setdefault(pid, []).append((((imgs[i].float() / 255.0) - mean) / std, pid))
        return src

    # The random part of the reference's own train-time transform (datasets/image_augmentation.py: ToTensor ->
    # Normalize -> [RandomHorizontalFlip -> RandomErasing(p)] -> Resize): the in-memory splits are already normalised
    # tensors of the target size, so the reference's RandomHorizontalFlip / RandomErasing instances are applied per
    # sample, exactly where its DataLoader would apply them. Both arms therefore train on augmented crops.
    from datasets import augmentations as ref_augmentations
    import torchvision.transforms as T
    aug = exp["task_opts"]["augment_opts"]
    ref_compose = ref_augmentations[aug["level"]](size=aug["img_size"], mean=aug["norm_mean"], std=aug["norm_std"])
    random_part = [t for t in ref_compose.transforms if isinstance(t, (T.RandomHorizontalFlip, T.RandomErasing))]
    train_transform = T.Compose(random_part) if random_part else None

    class _Split(ReIDImageDataset):
        flpr_transform = None

        def __getitem__(self, index):
            data, person_id, class_index = super().__getitem__(index)
            if self.flpr_transform is not None:
                data = self.flpr_transform(data)
            return data, person_id, class_index

    server = parser_server(exp, common)
    clients = parser_clients(exp, common)
    for c in clients:
        c.task_pipeline = _MemoryPipeline(c.task_pipeline.task_list, exp["task_opts"], make_split, DataLoader, _Split)
        c.task_pipeline.train_transform = train_transform
    stage = ExperimentStage(common, [exp])
    log = ExperimentLog(os.path.join(common["logs_dir"], "reference-bench.json"))

    def sync():
        for d in range(a.gpus if not a.cpu_debug else 0):
            torch.cuda.synchronize(d)

    import signal

    state = {"r": 0, "t_first": None, "t0": None, "stamps": [], "done": False}
    sampler = ClockSampler(0) if not a.cpu_debug else None

    def result(partial: bool) -> dict:
        """The JSON line from whatever has been measured so far (``partial``: the run was cut short by SIGTERM - the
        rounds completed inside the timed region, or, if it never got there, the warm-up rounds after the first)."""
        stamps = state["stamps"]
        timed = [t for t in stamps if state["t0"] is not None and t > state["t0"]]
        if timed:
            steps, ms = len(timed), (timed[-1] - state["t0"]) * 1e3
        elif len(stamps) >= 2:
            steps, ms = len(stamps) - 1, (stamps[-1] - stamps[0]) * 1e3
        else:
            return _unavailable("terminated before two rounds completed")
        clocks = sampler.stop() if sampler else None
        imgs = a.clients * a.images * a.epochs
        ms_per_step = ms / steps
        value = imgs / (ms_per_step / 1e3)
        h2d = a.clients * a.epochs * (2 * a.images) * 3 * a.height * a.width * 4
        cfg = bench_config(a, "reference", "") if bench_config else {}
        out = {
            "metric": metric, "value": round(value, 2), "unit": "images/s", "n_gpus": a.gpus, "steps": steps,
            "warmup": a.warmup, "ms_per_step": round(ms_per_step, 3), "higher_is_better": True, "scaling": "strong",
            "vs_baseline": None, "dtype": "fp32 (the reference has no mixed-precision path; cuDNN convolutions run "
                                          "TF32 under torch's defaults)",
            "data": "synthetic 256x128 crops (pre-normalised float tensors in host memory), random-init weights",
            "impl": "reference", "config": cfg,
            "notes": {"parallelism": f"reference thread-pool over device list cuda:0..{a.gpus - 1}",
                      "timing": "wall clock bracketed by cudaDeviceSynchronize on every device (the reference syncs "
                                "the host twice per training step, so wall == device time)"},
            "e2e": {"value": round(value, 2), "unit": "images/s", "ms_per_step": round(ms_per_step, 3),
                    "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": None},
            "gpu_launches": 0, "clocks": clocks,
            "convergence": convergence_block(log.records, state["r"]) if convergence_block else None,
        }
        if partial:
            out["partial"] = True
            out["steps_requested"] = a.steps
            out["partial_region"] = "timed" if timed else "warmup (first round excluded)"
        return out

    def on_term(signum, frame):                     # the driver's per-run limit: report what was measured so far
        if state["done"]:
            return
        state["done"] = True
        try:
            print(json.dumps(result(True)), flush=True)
        finally:
            os._exit(0)

    if rank == 0:
        try:
            signal.signal(signal.SIGTERM, on_term)
        except ValueError:                              # not the main thread
            pass

    # Own time budget (FLPR_REF_BUDGET_S, default 780 s from process start): the reference needs ~50 s per round, the
    # driver's per-run limit ended round 1's scaling runs (25 rounds) without a line. Past the budget - and with at
    # least two timed rounds measured - the arm stops and reports what it has, flagged ``partial`` like a SIGTERM.
    budget = float(os.environ.get("FLPR_REF_BUDGET_S", "780"))
    t_start = _T_IMPORT

    def over_budget() -> bool:
        return budget > 0 and time.perf_counter() - t_start > budget

    for _ in range(a.warmup):
        state["r"] += 1
        stage._process_one_round(state["r"], server, clients, exp, log)
        sync()
        state["stamps"].append(time.perf_counter())
        cleanup_payloads(common["checkpoints_dir"])
        if over_budget() and len(state["stamps"]) >= 3:
            break
    if sampler:
        sampler.start()
    sync()
    cut = over_budget() and len(state["stamps"]) >= 3
    if not cut:
        state["t0"] = time.perf_counter()
        for i in range(a.steps):
            state["r"] += 1
            stage._process_one_round(state["r"], server, clients, exp, log)
            sync()
            state["stamps"].append(time.perf_counter())
            if over_budget() and i + 1 >= 2 and i + 1 < a.steps:
                cut = True
                break
    state["done"] = True
    out = result(cut)
    if cut:
        out["partial_reason"] = f"own time budget of {budget:.0f} s (FLPR_REF_BUDGET_S)"
    cleanup_payloads(common["checkpoints_dir"])
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()
    return out

"""Experiment runtime (``experiment.py`` of the reference): ``ExperimentStage`` context manager + ``run()``,
``VirtualContainer`` device-slot allocator, ``ExperimentLog`` (re-exported).

Execution model: SPMD. One process per GPU (``torchrun``), clients round-robined over ranks, the *server* is a role
replicated on every rank whose aggregation / dispatch are collectives of :class:`flpr_b200.parallel.comm.FedComm`.
With a single process (``world_size == 1``) all clients live in this process, which is also the CPU plumbing mode.

The communication round is the reference's (``experiment.py:183-243``): sample online clients -> dispatch (integrated
on first contact, incremental afterwards) -> local training -> validation every ``val_interval`` rounds -> uploads ->
``server.calculate()``; payload checkpoints ``{round}-{src}-{dst}.ckpt`` are written by a background thread.
Every phase is timed on the device (CUDA events, max over ranks is taken by the caller) and recorded under
``perf`` in the experiment log, together with the bytes moved by the collectives.
"""
from __future__ import annotations

import os
import random
import threading
from contextlib import contextmanager
from datetime import datetime
from typing import Any, Dict, List, Optional, Sequence, Tuple, Union

import torch
import torch.distributed as dist

from ..methods import methods
from ..methods.fedbase import strip_private
from ..parallel.comm import FedComm
from ..utils.logger import Logger
from ..utils.misc import DeviceTimer, clear_cache, same_seeds
from .builder import parser_clients, parser_server
from . import resume
from .checkpoint import CheckpointStore
from .explog import ExperimentLog

__all__ = ["ExperimentStage", "ExperimentLog", "VirtualContainer"]


class VirtualContainer:
    """Device-slot allocator (``experiment.py:58-99``): ``{device: parallel}`` slots, ``possess_device(count)``.

    Race-free re-implementation: a condition variable guards the counters, a request larger than a device's capacity
    is clamped (the reference lets counters go negative and may hand out ``device=None``)."""

    def __init__(self, devices: Sequence[str], parallel: int = 1) -> None:
        self._cv = threading.Condition()
        self.capacity = {d: int(parallel) for d in devices}
        self.devices = dict(self.capacity)

    def max_worker(self) -> int:
        return sum(self.capacity.values())

    def acquire_device(self, count: int = 1) -> str:
        with self._cv:
            while True:
                for dev, free in self.devices.items():
                    need = min(count, self.capacity[dev])
                    if free >= need:
                        self.devices[dev] -= need
                        return dev
                self._cv.wait()

    def release_device(self, device: str, count: int = 1) -> None:
        with self._cv:
            self.devices[device] = min(self.capacity[device], self.devices[device] + min(count, self.capacity[device]))
            self._cv.notify_all()

    @contextmanager
    def possess_device(self, count: int = 1):
        dev = self.acquire_device(count)
        try:
            yield dev
        finally:
            self.release_device(dev, count)


def _dist_env() -> Tuple[int, int, int]:
    return (int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")),
            int(os.environ.get("LOCAL_RANK", "0")))


class ExperimentStage:
    def __init__(self, common_config: Dict, exp_configs: Union[Dict, Sequence[Dict]], source_factory=None):
        self.common_config = common_config
        self.exp_configs = [exp_configs] if isinstance(exp_configs, dict) else list(exp_configs)
        self.rank, self.world, self.local_rank = _dist_env()
        self.logger = Logger("stage", self.rank if self.world > 1 else None)
        self.source_factory = source_factory
        self.device = self._pick_device()
        self.container = VirtualContainer([str(self.device)], self.common_config.get("parallel", 1))
        self._owns_pg = False
        self.last_perf: Dict[str, Any] = {}

    # ------------------------------------------------------------------ environment
    def _pick_device(self) -> torch.device:
        devices = self.common_config.get("device", ["cpu"])
        wants_cuda = any(str(d).startswith("cuda") for d in devices)
        if wants_cuda and torch.cuda.is_available():
            if self.world > 1:
                return torch.device("cuda", self.local_rank % torch.cuda.device_count())
            first = next(str(d) for d in devices if str(d).startswith("cuda"))
            n_cuda = len({str(d) for d in devices if str(d).startswith("cuda")})
            if n_cuda > 1:
                # the reference spreads client threads over every listed device inside one process; this engine is
                # one process per GPU
                self.logger.warn(f"{n_cuda} CUDA devices are configured but WORLD_SIZE is 1: only {first} is used. "
                                 f"Launch with `torchrun --nproc-per-node {n_cuda} main.py ...` to use all of them.")
            return torch.device(first if ":" in first else "cuda:0")
        return torch.device("cpu")

    def __enter__(self):
        self.check_environment()
        return self

    def __exit__(self, exc_type, value, trace):
        pool = getattr(self, "_pool", None)
        if pool is not None:
            pool.shutdown(wait=False)
            self._pool = None
        if self._owns_pg and dist.is_initialized():
            dist.destroy_process_group()
        if exc_type is not None and issubclass(exc_type, Exception):
            self.logger.error(value)
        return False                                   # re-raise the original exception (reference bug fixed)

    def check_environment(self) -> None:
        try:
            torch.zeros(1).to(self.device)
        except Exception as ex:  # pragma: no cover
            self.logger.error(f"Not available for given device {self.device}:{ex}")
            raise SystemExit(1)
        if self.device.type == "cuda":
            torch.cuda.set_device(self.device)
        if self.world > 1 and not dist.is_initialized():
            backend = "nccl" if self.device.type == "cuda" else "gloo"
            kw = {"device_id": self.device} if backend == "nccl" else {}
            dist.init_process_group(backend, **kw)
            self._owns_pg = True
        datasets_dir = self.common_config["datasets_dir"]
        if self.source_factory is None and not os.path.exists(datasets_dir):
            self.logger.error(f"Datasets base directory could not be found with {datasets_dir}.")
            raise SystemExit(1)
        if os.path.exists(self.common_config["checkpoints_dir"]):
            self.logger.warn(f"Checkpoint directory {self.common_config['checkpoints_dir']} is not empty.")
        self.logger.info("Experiment stage build success.")

    # ------------------------------------------------------------------ one experiment
    def build(self, exp_config: Dict):
        """Construct comm, checkpoint store, server replica and the local clients for ``exp_config``."""
        eng = exp_config["engine_opts"]
        names = [c["client_name"] for c in exp_config["clients"]]
        n_local = len([i for i in range(len(names)) if i % self.world == self.rank])
        store_kw = dict(asynchronous=eng.get("async_checkpoint", True) and self.device.type == "cuda",
                        enabled=eng.get("checkpoints", True),
                        workers=eng.get("ckpt_workers") or min(16, max(8, 2 * n_local)),
                        arena_bytes=int(float(eng.get("ckpt_arena_gb") or min(8.0, max(3.0, 1.5 * n_local))) * (1 << 30)))
        ckpt_root = os.path.join(self.common_config["checkpoints_dir"], exp_config["exp_name"])
        if eng.get("mapped_checkpoints", True) and self.device.type == "cuda" and store_kw["asynchronous"]:
            # checkpoint files are CUDA-registered mappings, a snapshot is a set of DMAs into the file (tmpfs only;
            # other file systems keep the staged writer pipeline)
            from .mapped_store import MappedCheckpointStore
            os.makedirs(ckpt_root, exist_ok=True)
            store = MappedCheckpointStore(ckpt_root, payload_ring=int(eng.get("payload_ring", 0) or 0), **store_kw)
        else:
            store = CheckpointStore(ckpt_root, **store_kw)
        server = parser_server(exp_config, self.common_config, self.device, store)
        clients = parser_clients(exp_config, self.common_config, self.device, store, None, self.rank, self.world,
                                 self.source_factory)
        comm = None
        client_cls = methods[exp_config["exp_method"]].Client
        if hasattr(client_cls, "declare_buffers"):
            need = self._arena_bytes(server, len(names), exp_config)
            comm = FedComm(self.device, len(names), arena_bytes=need, mode=eng.get("comm_mode"),
                           timeout_s=eng.get("comm_timeout_s", 60.0))
            c_, h_, w_ = self._proto_shape(server, exp_config)
            client_cls.declare_buffers(comm, server.model, c_ * h_ * w_)
            for c in clients:
                c.comm = comm
            server.comm = comm
        for cid, name in enumerate(names):
            if hasattr(server, "bind_client"):
                local = next((c for c in clients if c.client_name == name), None)
                try:
                    server.bind_client(name, cid, local)
                except TypeError:
                    server.bind_client(name, cid)
        return store, comm, server, clients, names

    def _proto_shape(self, server, exp_config) -> Tuple[int, int, int]:
        net = server.model.net
        size = exp_config["task_opts"]["augment_opts"]["img_size"]
        if hasattr(net, "prototype_shape"):
            return net.prototype_shape(size)
        return (3, int(size[0]), int(size[1]))

    def _arena_bytes(self, server, n_clients: int, exp_config) -> int:
        mb = exp_config["engine_opts"].get("arena_mb", 0)
        if mb:
            return int(mb) << 20
        slots = (n_clients + self.world - 1) // self.world
        n = server.model.arena.numel
        c, h, w = self._proto_shape(server, exp_config)
        per_client = 2 * n * 4 + c * h * w * 4 + 64          # upload (+fisher) + token + counters
        return int(slots * per_client + 5 * n * 4 + (8 << 20))

    def run(self) -> None:
        for exp_config in self.exp_configs:
            self.run_experiment(exp_config)

    def run_experiment(self, exp_config: Dict) -> ExperimentLog:
        self._check_re_ranking(exp_config)
        same_seeds(exp_config["random_seed"])
        format_time = datetime.now().strftime("%Y-%m-%d-%H-%M")
        log = ExperimentLog(os.path.join(self.common_config["logs_dir"], f"{exp_config['exp_name']}-{format_time}.json"),
                            enabled=self.rank == 0)
        log.record("config", exp_config)
        self.logger.info(f"Experiment loading succeed: {exp_config['exp_name']}")
        self.logger.info(f"For more details: {log.save_path}")
        store, comm, server, clients, names = self.build(exp_config)
        timer = DeviceTimer(self.device)
        try:
            eng = exp_config["engine_opts"]
            # the newest manifest committed on EVERY rank (collective: all ranks take the same branch below, also after
            # an elastic restart in which some rank died before it could commit anything)
            resumed = resume.agreed_round(self, store) if eng.get("resume") else 0
            if eng.get("val_at_round0", True) and not resumed:
                self._validate_all(clients, names, exp_config, log, 0)   # initial validation (experiment.py:163-173)
            comm_rounds = int(exp_config["exp_opts"]["comm_rounds"])
            first_round = 1
            if resumed:
                first_round = resume.load(self, store, server, clients, comm, resumed) + 1
                self.logger.info(f"Resumed from the manifest of round {first_round - 1}.")
            interval = int(eng.get("resume_interval", 0) or 0)
            for curr_round in range(first_round, comm_rounds + 1):
                self.logger.info(f"Start communication round: {curr_round:0>3d}/{comm_rounds:0>3d}")
                self._process_one_round(curr_round, server, clients, names, exp_config, log, timer, comm)
                resume.maybe_inject_fault(self, curr_round, "round")
                if interval and curr_round % interval == 0:
                    if self.device.type == "cuda":
                        self._join_deferred_aggregate()          # the manifest snapshots the server replica
                    resume.save(self, store, curr_round, server, clients, comm)
            self._gather_logs(log)
        finally:
            if self.device.type == "cuda":
                self._join_deferred_aggregate()
            store.flush()
            store.close()
            perf = {k: sum(v) for k, v in timer.flush().items()}
            if comm is not None:
                perf["comm_bytes"] = comm.bytes_moved
                comm.check_errors()
                comm.close()
            self.last_perf = perf
            log.record("perf", {f"rank{self.rank}": perf}, flush=True)
            log.close()
        del server, clients
        clear_cache()
        return log

    # ------------------------------------------------------------------ one round
    def _process_one_round(self, curr_round, server, clients, names, exp_config, log, timer, comm) -> None:
        eng = exp_config["engine_opts"]
        save_payloads = eng.get("save_payload_ckpts", True)
        local = {c.client_name: c for c in clients}
        online = random.sample(names, exp_config["exp_opts"]["online_clients"])
        val_interval = exp_config["exp_opts"]["val_interval"]
        federated = getattr(type(server), "federated", None)
        if federated is None:
            federated = hasattr(server, "uploaded")

        store = getattr(server, "store", None)
        if store is not None:
            every = max(1, int(eng.get("checkpoint_interval", 1) or 1))
            store.muted = (curr_round % every) != 0
        if self.device.type == "cuda" and store is not None:
            store.fence()                 # snapshot DMAs of the previous round precede any overwrite of their sources
        if comm is not None:
            comm.poll_errors()

        # ---- server -> clients ------------------------------------------------------------------------------------
        with timer("dispatch"):
            first = [n for n in online if n not in server.clients]
            if first:
                self._join_deferred_aggregate()      # a first-contact dispatch reads the server replica
            for n in first:
                server.register_client(n)
            if hasattr(server, "prepare_dispatch"):
                server.prepare_dispatch(online, first)
            for n in online:
                client = local.get(n)
                if client is None:
                    continue
                if n in first:
                    state = server.get_dispatch_integrated_state(n)
                    if state is not None:
                        client.update_by_integrated_state(state)
                else:
                    state = server.get_dispatch_incremental_state(n)
                    if state is not None:
                        client.update_by_incremental_state(state)
                if save_payloads:
                    server.save_state(f"{curr_round}-{server.server_name}-{n}", strip_private(state), True)
                del state

        # ---- local training ---------------------------------------------------------------------------------------
        with timer("train"):
            todo = [local[n] for n in online if n in local]
            workers = min(self.container.max_worker(), len(todo))
            if workers > 1 and self.device.type == "cuda" and eng.get("client_threads", True) and \
                    all(getattr(c.model.net, "thread_safe_rng", False) for c in todo):
                self._train_parallel(todo, log, curr_round, workers)
            elif workers > 1 and self.device.type == "cpu" and eng.get("client_threads") == "force":
                self._train_parallel_cpu(todo, log, curr_round, workers)
            else:
                for client in todo:
                    self._process_train(client, log, curr_round, self.container)

        # ---- validation -------------------------------------------------------------------------------------------
        if curr_round % val_interval == 0:
            with timer("validate"):
                self._validate_all(clients, names, exp_config, log, curr_round)

        # ---- clients -> server ------------------------------------------------------------------------------------
        self._join_deferred_aggregate()              # last round's deferred mean has read the upload slots
        with timer("upload"):
            for n in online:
                client = local.get(n)
                if client is not None:
                    state = client.get_incremental_state()
                    if save_payloads:
                        client.save_state(f"{curr_round}-{n}-{server.server_name}", strip_private(state), True)
                    if state is not None:
                        server.set_client_incremental_state(n, state)
                    del state
                elif federated:
                    server.set_client_incremental_state(n, None)      # slot lives on another rank
        with timer("aggregate"):
            if store is not None and self.device.type == "cuda":
                # calculate() overwrites the server replica in place: snapshots staged from live views of it (dispatch
                # payloads, the server model) must have left the device first; client snapshots keep streaming
                store.fence(server.name)
            overlap = (eng.get("overlap_aggregate", True) and self.device.type == "cuda" and comm is not None
                       and getattr(comm, "mode", "") == "p2p" and getattr(server, "split_calculate", False))
            if overlap:
                # BASELINE.json: "federated rounds overlap aggregation with the next client's local step on CUDA
                # streams". The part of the aggregation the next dispatch depends on stays here; the bulk runs on the
                # communication stream (flag channel 1) next to the next round's mix / prototype pass / training.
                server.calculate_urgent()
                cs = self._comm_stream()
                main = torch.cuda.current_stream(self.device)
                cs.wait_stream(main)
                with torch.cuda.stream(cs):
                    comm.set_channel(1)
                    comm.block_cap = int(eng.get("overlap_comm_blocks", 24))   # a small grid: its blocks spin at the
                    try:                                                        # barriers while a peer is late, and they
                        server.calculate_deferred()                             # share the SMs with the training kernels
                    finally:
                        comm.block_cap = 0
                        comm.set_channel(0)
                    ev = torch.cuda.Event()
                    ev.record(cs)
                self._agg_event = ev
            else:
                server.calculate()
        if comm is not None:
            comm.poll_errors()            # a missed barrier surfaces in the round it happened, not at the very end
        log.flush()

    def _validate_all(self, clients, names, exp_config, log, curr_round: int) -> None:
        """Validation of every client on every task (``experiment.py:163-173, :218-229``). Default: each rank validates
        the clients it hosts. ``engine_opts.sharded_validation`` (world > 1): all ranks walk the global (client, task)
        list together and rank every gallery in ``1 / world`` slices (``evaluation/sharded.py``)."""
        eng = exp_config["engine_opts"]
        if not (eng.get("sharded_validation", False) and self.world > 1):
            for client in clients:
                self._process_val(client, log, curr_round, self.container)
            return
        from ..evaluation.sharded import ShardedRanker
        ranker = getattr(self, "_ranker_obj", None)
        if ranker is None:
            ranker = self._ranker_obj = ShardedRanker(self.device)
        local = {c.client_name: c for c in clients}
        for cid, cfg in enumerate(exp_config["clients"]):
            client = local.get(cfg["client_name"])
            if client is not None:
                client._ranker = ranker
                try:
                    self._process_val(client, log, curr_round, self.container)
                finally:
                    client._ranker = None
            else:
                for _ in range(len(cfg["tasks"])):                   # one collective per task of that client
                    ranker.participate(cid % self.world)

    def _check_re_ranking(self, exp_config: Dict) -> None:
        """``engine_opts.re_ranking`` needs the gallery-to-gallery neighbourhoods of the WHOLE gallery, which the
        gallery-sharded validation never holds on one rank: refuse the combination instead of skipping re-ranking."""
        from ..ops.rank import re_ranking_params
        eng = exp_config["engine_opts"]
        rr = re_ranking_params(eng.get("re_ranking", False))
        if rr is not None and eng.get("sharded_validation", False) and self.world > 1:
            raise ValueError("engine_opts.re_ranking cannot be combined with engine_opts.sharded_validation on "
                             f"{self.world} ranks: re-ranking needs the neighbourhoods of the whole gallery on one rank. "
                             "Turn one of the two off.")

    def _comm_stream(self):
        st = getattr(self, "_comm_stream_obj", None)
        if st is None:
            from ..ops import native
            st = self._comm_stream_obj = native.dedicated_stream(self.device, priority=-1)
        return st

    def _join_deferred_aggregate(self) -> None:
        """Make the compute stream wait for an aggregation that is still running on the communication stream."""
        ev = getattr(self, "_agg_event", None)
        if ev is not None:
            torch.cuda.current_stream(self.device).wait_event(ev)
            self._agg_event = None

    def _train_parallel(self, todo, log, curr_round: int, workers: int) -> None:
        """``parallel`` clients per device train concurrently (the reference's thread pool, ``experiment.py:206-216``),
        each on its own CUDA stream: while one client's thread waits for its epoch result (the early-stopping rule
        needs loss / accuracy on the host) the other threads keep the GPU fed."""
        from concurrent.futures import ThreadPoolExecutor
        dev = self.device
        main = torch.cuda.current_stream(dev)
        start = torch.cuda.Event()
        start.record(main)
        done: List[torch.cuda.Event] = []

        def run(client) -> None:
            from ..ops import native
            native.register_client_thread()
            torch.cuda.set_device(dev)
            stream = getattr(client, "_stream", None)
            if stream is None:
                stream = client._stream = native.dedicated_stream(dev)
            with torch.cuda.stream(stream):
                stream.wait_event(start)
                self._process_train(client, log, curr_round, self.container)
                ev = torch.cuda.Event()
                ev.record(stream)
            done.append(ev)

        pool = getattr(self, "_pool", None)
        if pool is None or getattr(self, "_pool_workers", 0) != workers:
            if pool is not None:
                pool.shutdown(wait=True)
            pool = self._pool = ThreadPoolExecutor(max_workers=workers, thread_name_prefix="flpr-client")
            self._pool_workers = workers
        futures = [pool.submit(run, c) for c in todo]
        err = None
        for f in futures:
            try:
                f.result(timeout=1800)
            except Exception as ex:  # noqa: BLE001
                err = err or ex
        for ev in done:
            main.wait_event(ev)
        if err is not None:
            raise err

    def _train_parallel_cpu(self, todo, log, curr_round: int, workers: int) -> None:
        """CPU twin of :meth:`_train_parallel` (``engine_opts.client_threads: force``): the same thread pool without
        streams - used by the CPU test-suite to exercise the thread-safety of the client path."""
        from concurrent.futures import ThreadPoolExecutor
        with ThreadPoolExecutor(max_workers=workers, thread_name_prefix="flpr-client") as pool:
            futures = [pool.submit(self._process_train, c, log, curr_round, self.container) for c in todo]
            err = None
            for f in futures:
                try:
                    f.result(timeout=1800)
                except Exception as ex:  # noqa: BLE001
                    err = err or ex
        if err is not None:
            raise err

    def _gather_logs(self, log: ExperimentLog) -> None:
        """C7: metrics of remote clients are gathered to rank 0, which owns the JSON file."""
        if self.world > 1:
            parts: List[Optional[dict]] = [None] * self.world if self.rank == 0 else None
            dist.gather_object(log.records.get("data", {}), parts, dst=0)
            if self.rank == 0:
                for p in parts[1:]:
                    log.merge({"data": p})

    @staticmethod
    def _process_train(client, log, curr_round, container) -> None:
        with container.possess_device() as device:
            try:
                task = client.task_pipeline.next_task()
                if task["tr_epochs"] != 0:
                    out = client.train(epochs=task["tr_epochs"], task_name=task["task_name"],
                                       tr_loader=task["tr_loader"], val_loader=task["query_loader"], device=device)
                    log.record(f"data.{client.client_name}.{curr_round}.{task['task_name']}",
                               {"tr_acc": out["accuracy"], "tr_loss": out["loss"]})
            except Exception as ex:
                client.logger.error(ex)
                raise

    @staticmethod
    def _process_val(client, log, curr_round, container) -> None:
        with container.possess_device(container.max_worker()) as device:
            try:
                pipeline = client.task_pipeline
                for tid in range(len(pipeline.task_list)):
                    task = pipeline.get_task(tid)
                    out = client.validate(task_name=task["task_name"], query_loader=task["query_loader"],
                                          gallery_loader=task["gallery_loaders"], device=device)
                    cmc, mAP = out[0], out[1]
                    r = lambda c, k: float(c[k]) if len(c) > k else float(c[-1])  # noqa: E731
                    rec = {"val_rank_1": r(cmc, 0), "val_rank_3": r(cmc, 2), "val_rank_5": r(cmc, 4),
                           "val_rank_10": r(cmc, 9), "val_map": float(mAP)}
                    if len(out) > 3:                   # engine_opts.re_ranking: the re-ranked (cmc, mAP)
                        rr_cmc, rr_map = out[3]
                        rec.update({"val_rr_rank_1": r(rr_cmc, 0), "val_rr_rank_3": r(rr_cmc, 2),
                                    "val_rr_rank_5": r(rr_cmc, 4), "val_rr_rank_10": r(rr_cmc, 9),
                                    "val_rr_map": float(rr_map)})
                    log.record(f"data.{client.client_name}.{curr_round}.{task['task_name']}", rec)
            except Exception as ex:
                client.logger.error(ex)
                raise

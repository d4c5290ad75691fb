"""Two or more ranks with a robust aggregator (``server: aggregator: median``) and one Byzantine client: the server role
is replicated, and after 3 rounds every rank's server replica must be bit-identical and finite.

    FLPR_TMP=/tmp/x torchrun --standalone --local-addr 127.0.0.1 --nproc-per-node 2 \
        tests/dist_robust_agg_check.py cpu          # gloo
    FLPR_TMP=/tmp/x torchrun ... tests/dist_robust_agg_check.py cuda 0|1    # peer-memory collectives, NVLS off / on

client-0 uploads 1e30 / NaN (overwritten in its slot after the upload). Rank 0 saves its replica to
``$FLPR_TMP/robust_rank0.pt`` and every rank writes its payload checkpoints under ``$FLPR_TMP/r{rank}`` (the caller
replays the median from them)."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from flpr_b200.runtime.experiment import ExperimentStage  # noqa: E402
from helpers import tiny_common, tiny_experiment, tiny_factory  # noqa: E402

AGGREGATOR = {"name": "median"}
N_CLIENTS = 3


def poison():
    from flpr_b200.methods.fedbase import FedClient
    inner = FedClient.get_incremental_state

    def poisoned(self, **kw):
        st = inner(self, **kw)
        if self.client_name == "client-0":
            slot = self.comm.client_view("up", self.client_id)
            slot[0::3] = 1e30
            slot[1::3] = float("nan")
        return st
    FedClient.get_incremental_state = poisoned


def main():
    device = sys.argv[1] if len(sys.argv) > 1 else "cpu"
    nvls = (sys.argv[2] != "0") if len(sys.argv) > 2 else True
    base = os.environ.get("FLPR_TMP", "/tmp/flpr_dist")
    rank = int(os.environ.get("RANK", "0"))
    tmp = os.path.join(base, f"r{rank}")
    common = tiny_common(tmp, device=device)
    common["defaults"]["exp_opts"]["comm_rounds"] = 3
    common["defaults"]["exp_opts"]["online_clients"] = N_CLIENTS
    factory = tiny_factory()
    if device != "cpu":
        from flpr_b200.data.synthetic import synthetic_source_factory
        common["defaults"]["task_opts"]["augment_opts"]["img_size"] = [64, 32]
        common["defaults"]["task_opts"]["loader_opts"]["batch_size"] = 8
        factory = synthetic_source_factory(num_ids=4, train_per_id=4, size=(64, 32))
    cfg = tiny_experiment(common, "fedavg", n_clients=N_CLIENTS, n_tasks=1)
    cfg["server"]["aggregator"] = dict(AGGREGATOR)
    poison()
    from flpr_b200.runtime.explog import ExperimentLog
    from flpr_b200.utils.misc import DeviceTimer, same_seeds
    with ExperimentStage(common, [cfg], source_factory=factory) as stage:
        same_seeds(cfg["random_seed"])                 # before the build: every rank initialises the same replica
        store, comm, server, clients, names = stage.build(cfg)
        assert comm.world >= 2 and comm.mode == ("gloo" if device == "cpu" else "p2p"), (comm.world, comm.mode)
        comm.nvls = nvls
        log = ExperimentLog(os.path.join(tmp, "log.json"), enabled=False)
        timer = DeviceTimer(stage.device)
        for r in (1, 2, 3):
            stage._process_one_round(r, server, clients, names, cfg, log, timer, comm)
        store.flush()
        n = comm.rank_view("glob").numel()
        mine = server.model.arena.master[:n].clone()
        gathered = [torch.empty_like(mine) for _ in range(comm.world)]
        dist.all_gather(gathered, mine)
        same = all(torch.equal(gathered[0], g) for g in gathered[1:])
        finite = bool(torch.isfinite(mine).all())
        no_nvls = getattr(comm, "nvls_launches", 0) == 0
        if stage.rank == 0:
            a = server.model.arena
            torch.save({"x": {"net." + k: a.view(mine, k).flatten().cpu() for k, seg in a.segments.items()
                              if seg.offset + seg.numel <= n}},
                       os.path.join(base, "robust_rank0.pt"))
        store.close()
    if stage.rank == 0:
        ok = same and finite and no_nvls
        print("DIST_ROBUST_AGG", "OK" if ok else "FAILED", f"identical={same} finite={finite} no_nvls={no_nvls}",
              flush=True)


if __name__ == "__main__":
    main()

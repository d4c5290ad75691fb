"""Two or more ranks with a server optimizer (``server: server_opt: adam``): the server role is replicated, and after
3 rounds every rank's server replica and its moments ``m`` / ``v`` must be bit-identical - the step runs on the
bitwise-identical aggregated mean on every rank, no extra communication keeps them in sync.

    FLPR_TMP=/tmp/x torchrun --standalone --local-addr 127.0.0.1 --nproc-per-node 2 \
        tests/dist_server_opt_check.py cpu          # gloo
    FLPR_TMP=/tmp/x torchrun ... tests/dist_server_opt_check.py cuda 0|1    # peer-memory collectives, NVLS off / on

Rank 0 saves its replica, ``m``, ``v`` to ``$FLPR_TMP/server_opt_rank0.pt`` and every rank writes its payload
checkpoints under ``$FLPR_TMP/r{rank}`` (the caller replays the server step from them)."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from flpr_b200.runtime.experiment import ExperimentStage  # noqa: E402
from helpers import tiny_common, tiny_experiment, tiny_factory  # noqa: E402

SERVER_OPT = {"name": "adam", "lr": 0.01, "beta1": 0.9, "beta2": 0.99, "tau": 1e-3}


def main():
    device = sys.argv[1] if len(sys.argv) > 1 else "cpu"
    nvls = (sys.argv[2] != "0") if len(sys.argv) > 2 else True
    base = os.environ.get("FLPR_TMP", "/tmp/flpr_dist")
    rank = int(os.environ.get("RANK", "0"))
    tmp = os.path.join(base, f"r{rank}")
    common = tiny_common(tmp, device=device)
    common["defaults"]["exp_opts"]["comm_rounds"] = 3
    factory = tiny_factory()
    if device != "cpu":
        from flpr_b200.data.synthetic import synthetic_source_factory
        common["defaults"]["task_opts"]["augment_opts"]["img_size"] = [64, 32]
        common["defaults"]["task_opts"]["loader_opts"]["batch_size"] = 8
        factory = synthetic_source_factory(num_ids=4, train_per_id=4, size=(64, 32))
    cfg = tiny_experiment(common, "fedavg", n_clients=2, n_tasks=1)
    cfg["server"]["server_opt"] = dict(SERVER_OPT)
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
        mine = [server.model.arena.master[:n].clone(), server.opt_m.clone(), server.opt_v.clone()]
        same = True
        for t in mine:
            gathered = [torch.empty_like(t) for _ in range(comm.world)]
            dist.all_gather(gathered, t)
            same = same and all(torch.equal(gathered[0], g) for g in gathered[1:])
        finite = all(bool(torch.isfinite(t).all()) for t in mine)
        if stage.rank == 0:
            a = server.model.arena

            def named(flat):                      # payload keys, standard layout
                return {"net." + k: a.view(flat, k).flatten().cpu() for k, seg in a.segments.items()
                        if seg.offset + seg.numel <= n}
            torch.save({"x": named(mine[0]), "m": named(mine[1]), "v": named(mine[2]),
                        "nvls_launches": getattr(comm, "nvls_launches", 0)},
                       os.path.join(base, "server_opt_rank0.pt"))
        store.close()
    if stage.rank == 0:
        print("DIST_SERVER_OPT", "OK" if (same and finite) else "FAILED", f"identical={same} finite={finite}",
              flush=True)


if __name__ == "__main__":
    main()

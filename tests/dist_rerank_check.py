"""Two-rank (gloo) check: ``engine_opts.sharded_validation`` together with ``engine_opts.re_ranking`` is refused with a
``ValueError`` at experiment start on every rank, before any training or validation runs."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from flpr_b200.runtime.experiment import ExperimentStage  # noqa: E402
from helpers import tiny_common, tiny_experiment, tiny_factory  # noqa: E402


def main():
    tmp = os.path.join(os.environ.get("FLPR_TMP", "/tmp/flpr_dist"), f"r{os.environ.get('RANK', '0')}")
    common = tiny_common(tmp)
    cfg = tiny_experiment(common, "fedavg", n_clients=2, n_tasks=1)
    cfg["engine_opts"].update(sharded_validation=True, re_ranking=True)
    msg = None
    with ExperimentStage(common, [cfg], source_factory=tiny_factory()) as stage:
        try:
            stage.run_experiment(cfg)
        except ValueError as ex:
            msg = str(ex)
        ok = msg is not None and "sharded_validation" in msg and stage.world == 2
    print("DIST_RERANK", "OK" if ok else "FAILED", msg, flush=True)


if __name__ == "__main__":
    main()

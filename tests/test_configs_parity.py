"""The shipped experiment configs carry the reference's values (SURVEY §2.1 "Config system": ``common.yaml`` + 46
experiment YAMLs). Compared file by file against the reference's configs, stored parsed in
``tests/golden/reference_configs.json.gz``."""
import gzip
import json
import os

import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OURS = os.path.join(ROOT, "configs")
with gzip.open(os.path.join(ROOT, "tests", "golden", "reference_configs.json.gz"), "rt") as _f:
    REF = json.load(_f)

# keys this engine adds on top of the reference's schema
EXTRA_KEYS = {"engine_opts"}


def _load(path):
    with open(path) as f:
        return yaml.load(f, Loader=yaml.Loader)


def _strip(d):
    return {k: v for k, v in d.items() if k not in EXTRA_KEYS} if isinstance(d, dict) else d


def _json(d):
    return json.loads(json.dumps(d))


def test_every_reference_experiment_yaml_has_an_identical_counterpart():
    assert len(REF["experiments"]) == 46
    for rel, ref in sorted(REF["experiments"].items()):
        mine = os.path.join(OURS, rel)
        assert os.path.exists(mine), f"missing config {rel}"
        assert _json(_strip(_load(mine))) == ref, rel


def test_common_defaults_match():
    ref, mine = _json(REF["common"]), _json(_load(os.path.join(OURS, "common.yaml")))
    # the one deliberate difference: the reference ships ``multiprocessing_context: spawn`` with ``num_workers: 0``, which
    # current PyTorch rejects with a ValueError (SURVEY §8 item 3); ours ships ``null``
    assert ref["defaults"]["task_opts"]["loader_opts"].pop("multiprocessing_context") == "spawn"
    assert mine["defaults"]["task_opts"]["loader_opts"].pop("multiprocessing_context") is None
    assert _strip(mine["defaults"]) == ref["defaults"]
    assert {k: v for k, v in mine.items() if k != "defaults"} == {k: v for k, v in ref.items() if k != "defaults"}


def test_batch_launcher_runs_the_reference_experiment_list():
    """``startup.sh`` (reference: ``startup.sh``): valid shell, launches ``main.py`` in the background with the same ten
    basis experiments in the same order, each of which exists here."""
    import re
    import subprocess
    mine = os.path.join(ROOT, "startup.sh")
    assert subprocess.run(["bash", "-n", mine]).returncode == 0

    def experiments(path):
        with open(path) as f:
            return [os.path.normpath(p) for p in re.findall(r"[\w./]*configs/[\w./]+\.yaml", f.read())]

    ours = experiments(mine)
    assert len(ours) == 10 and all(os.path.exists(os.path.join(ROOT, p)) for p in ours)
    assert ours == REF["startup_experiments"]
    with open(mine) as f:
        text = f.read()
    assert "main.py --experiments" in text and "nohup" in text and text.rstrip().endswith("&")

"""``bench.py`` prints ONE JSON line with the keys the driver reads (metric / value / e2e / gpu_launches / clocks ...).
Exercised through ``--cpu-debug`` (a tiny CPU experiment through the same harness: build_config -> ExperimentStage rounds
-> device-timed region -> end-to-end region -> JSON), so that a refactoring of the harness cannot break the contract
unnoticed between GPU sessions."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

REQUIRED = {"metric": str, "value": (int, float), "unit": str, "n_gpus": int, "steps": int, "warmup": int,
            "ms_per_step": (int, float), "higher_is_better": bool, "scaling": str, "dtype": str, "data": str,
            "config": dict, "e2e": dict, "gpu_launches": int}


def _run(*flags, timeout=900):
    env = dict(os.environ)
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), *flags], capture_output=True, text=True,
                       timeout=timeout, cwd=ROOT, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1, f"expected exactly one JSON line, got {len(lines)}"
    return json.loads(lines[0])


def test_bench_cpu_debug_prints_the_driver_contract():
    d = _run("--cpu-debug", "--steps", "1", "--warmup", "1")
    for key, ty in REQUIRED.items():
        assert key in d, f"missing key {key}"
        assert isinstance(d[key], ty), (key, type(d[key]))
    assert "vs_baseline" in d and "clocks" in d
    assert d["steps"] == 1 and d["warmup"] == 1 and d["n_gpus"] == 1 and d["higher_is_better"] is True
    assert d["scaling"] in ("strong", "weak") and d["impl"] == "flpr"
    assert d["value"] > 0 and d["ms_per_step"] > 0
    for key in ("value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"):
        assert key in d["e2e"], key
    assert d["e2e"]["value"] > 0
    for key in ("model", "method", "clients", "global_batch"):
        assert key in d["config"], key
    conv = d.get("convergence")
    assert conv and len(conv["tr_loss"]) == conv["rounds"] >= 2 and all(v == v for v in conv["tr_loss"])


def test_reference_arm_reports_itself_when_the_reference_is_missing(tmp_path):
    """``--impl reference`` without ``oracle/_ref`` must print ``{"impl": "reference", "unavailable": ...}`` and exit
    0 (driver contract). Checked on the arm's own function with the reference directory pointed elsewhere."""
    sys.path.insert(0, ROOT)
    from baseline import reference_arm as ra
    saved = ra.REF
    ra.REF = str(tmp_path / "nowhere")
    try:
        class A:
            cpu_debug, gpus = True, 1
        out = ra.run_reference_arm(A(), None, None, "m", None)
    finally:
        ra.REF = saved
    assert out["impl"] == "reference" and "unavailable" in out and "\n" not in out["unavailable"]


def test_reference_arm_runs_the_installed_reference():
    """``--impl reference --cpu-debug``: the unmodified reference in ``oracle/_ref`` driven through its own builder /
    ``ExperimentStage._process_one_round`` prints the same JSON line (``impl: reference``)."""
    import pytest
    if not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "methods")):
        pytest.skip("the reference oracle is not built in oracle/_ref")
    d = _run("--impl", "reference", "--cpu-debug", "--steps", "1", "--warmup", "1")
    assert d.get("impl") == "reference" and "unavailable" not in d
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "config"):
        assert key in d, key
    assert d["value"] > 0 and d["steps"] == 1


def test_bench_under_torchrun_prints_one_line_from_rank0():
    """The driver's multi-GPU launch form (``python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py
    --gpus N``) on the CPU debug path (gloo): the cross-rank reductions of the harness run, rank 0 alone prints the line."""
    env = dict(os.environ, OMP_NUM_THREADS="2")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    import socket
    with socket.socket() as sock:                        # a free port: a fixed one would collide with a parallel run
        sock.bind(("127.0.0.1", 0))
        port = sock.getsockname()[1]
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "bench.py"),
                        "--gpus", "2", "--steps", "1", "--warmup", "1", "--cpu-debug"], capture_output=True, text=True,
                       timeout=900, cwd=ROOT, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1, lines
    d = json.loads(lines[0])
    assert d["n_gpus"] == 2 and d["value"] > 0 and d["e2e"]["value"] > 0 and d["steps"] == 1

"""YAML configuration with the reference's semantics (``main.py:12-22``, SURVEY §5.6).

* ``common.yaml`` carries ``datasets_dir / checkpoints_dir / logs_dir / parallel / device`` and a ``defaults`` block.
* every experiment YAML is **shallow**-merged over ``defaults``: an experiment's ``model_opts`` block replaces the
  default block wholesale.
* unknown keys flow through untouched – they become ``**kwargs`` of nets / criteria / clients / servers.

New (optional) keys understood by this engine live under ``engine_opts`` (dtype, comm mode, reference-compat flags).
"""
from __future__ import annotations

import copy
import os
from typing import Any, Dict, List, Sequence

import yaml

ENGINE_DEFAULTS: Dict[str, Any] = {
    "compute_dtype": "bf16",          # bf16 tensor-core path on CUDA, fp32 on CPU
    "comm_mode": None,                # None -> p2p on CUDA, gloo/local on CPU; "nccl" = baseline harness
    "arena_mb": 0,                    # 0 -> sized automatically from the model
    "async_checkpoint": True,         # write payload / model checkpoints off the critical path
    "save_payload_ckpts": True,       # '{round}-{src}-{dst}.ckpt' files (experiment.py:199-202,235-238)
    "checkpoint_interval": 1,         # snapshot every N-th round (1 = every round, like the reference)
    "mapped_checkpoints": True,       # CUDA + RAM-disk checkpoints_dir: files are CUDA-registered mappings written by
                                      # DMA (runtime/mapped_store.py); False = staged writer-process pipeline
    "payload_ring": 0,                # keep only the last N rounds of '{round}-{src}-{dst}.ckpt' files, recycling the
                                      # mappings of older rounds (0 = keep every round, like the reference)
    "ckpt_workers": 0,                # writer processes (0 -> 8..16 by the number of local clients)
    "ckpt_arena_gb": 0,               # pinned staging arena (0 -> 3..8 GB by the number of local clients)
    "overlap_aggregate": True,        # methods with a deferred aggregation part (FedSTIL's 125 MB FedAvg mean into the
                                      # server replica) run it on a communication stream / second flag channel,
                                      # concurrently with the next round's mix and local training
    "overlap_comm_blocks": 24,        # grid of that overlapped collective (its blocks spin at the cross-rank barriers
                                      # next to the training kernels)
    "sharded_validation": False,      # world > 1: all ranks rank every client's gallery in 1/world slices
                                      # (evaluation/sharded.py) instead of each rank validating its own clients alone
    "re_ranking": False,              # also rank with k-reciprocal re-ranking (val_rr_* next to val_*): true = k1 20,
                                      # k2 6, lambda 0.3, or a dict {k1, k2, lambda_value}; not with sharded_validation
    "client_threads": True,           # `parallel` clients per device train concurrently on their own CUDA streams
    "resume": False,                  # continue from {checkpoints_dir}/{exp}/_resume/rank{r}.ckpt when present
    "resume_interval": 0,             # write the resume manifest every N rounds (0 = never)
    "device_augment": True,           # run flip / erasing / resize on the GPU
    "cache_prototypes": False,        # FedSTIL: recompute the frozen-trunk pass every epoch like the reference
    "reference_compat": True,         # reproduce documented reference quirks (SURVEY §7.5.5)
    "val_at_round0": True,
    "train_l1_anchor": None,          # FedSTIL: also train the L1 anchor like the reference's optimizer does (quirk,
                                      # fused into the optimizer kernel); None -> follows `reference_compat`
    "init_state": None,               # path of a {server/client name | "*": net state_dict} table loaded at build time
}


def load_yaml(path: str) -> Dict[str, Any]:
    with open(path, "r") as f:
        return yaml.load(f, Loader=yaml.Loader)


def load_common(path: str) -> Dict[str, Any]:
    common = load_yaml(path)
    if not isinstance(common.get("device", []), list):
        common["device"] = [common["device"]]
    common.setdefault("parallel", 1)
    common.setdefault("defaults", {})
    return common


def merge_experiment(common: Dict[str, Any], exp: Dict[str, Any]) -> Dict[str, Any]:
    """Shallow ``dict.update`` of the experiment over ``common['defaults']`` (``main.py:19-20``)."""
    cfg = dict(copy.deepcopy(common.get("defaults", {})))
    cfg.update(copy.deepcopy(exp))
    eng = dict(ENGINE_DEFAULTS)
    eng.update(cfg.get("engine_opts") or {})
    cfg["engine_opts"] = eng
    return cfg


def load_experiments(common_path: str, experiment_paths: Sequence[str]):
    common = load_common(common_path)
    exps: List[Dict[str, Any]] = [merge_experiment(common, load_yaml(p)) for p in experiment_paths]
    return common, exps


def resolve_dir(base: str, path: str) -> str:
    return path if os.path.isabs(path) else os.path.normpath(os.path.join(base, path))

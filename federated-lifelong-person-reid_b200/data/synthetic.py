"""Synthetic person-crop data (no dataset is available offline).

* :func:`make_array_split` – in-memory uint8 crops with identity-dependent structure (so that training actually
  learns and CMC/mAP are meaningful), used by tests and ``bench.py``.
* :func:`write_imagefolder_tree` – materialises the reference's on-disk layout
  ``{datasets_dir}/task-{c}-{t}/{train,query,gallery}/{pid}/*.jpg`` (``datasets/preprocessed_shuffle/README.md``).
"""
from __future__ import annotations

import os
from typing import Dict, Sequence, Tuple

import numpy as np
import torch

from .datasets import ArrayReIDDataset


def _identity_images(pid: int, count: int, size: Tuple[int, int], rng: np.random.Generator) -> np.ndarray:
    h, w = size
    base_rng = np.random.default_rng(10_007 * (pid + 1))
    coarse = base_rng.integers(0, 256, size=(8, 4, 3)).astype(np.float32)
    base = np.kron(coarse, np.ones((h // 8 + 1, w // 4 + 1, 1), dtype=np.float32))[:h, :w]
    noise = rng.normal(0.0, 24.0, size=(count, h, w, 3)).astype(np.float32)
    shift = rng.normal(0.0, 12.0, size=(count, 1, 1, 3)).astype(np.float32)
    return np.clip(base[None] + noise + shift, 0, 255).astype(np.uint8)


def make_array_split(person_ids: Sequence[int], per_id: int, size: Tuple[int, int] = (256, 128), seed: int = 0,
                     pin: bool = True) -> ArrayReIDDataset:
    rng = np.random.default_rng(seed)
    imgs, pids = [], []
    for pid in person_ids:
        imgs.append(_identity_images(int(pid), per_id, size, rng))
        pids += [int(pid)] * per_id
    images = torch.from_numpy(np.concatenate(imgs, 0)) if imgs else torch.zeros((0, *size, 3), dtype=torch.uint8)
    return ArrayReIDDataset(images, torch.tensor(pids, dtype=torch.long), classes=sorted(int(p) for p in person_ids),
                            pin=pin)


def random_array_split(n: int, num_ids: int, size: Tuple[int, int] = (256, 128), id_offset: int = 0, seed: int = 0,
                       pin: bool = True) -> ArrayReIDDataset:
    """Pure-noise crops (throughput benchmarking: content does not matter, shapes and label range do)."""
    g = torch.Generator().manual_seed(seed)
    images = torch.randint(0, 256, (n, size[0], size[1], 3), dtype=torch.uint8, generator=g)
    pids = torch.randint(0, num_ids, (n,), generator=g) + id_offset
    return ArrayReIDDataset(images, pids, pin=pin)


def synthetic_source_factory(num_ids: int = 8, train_per_id: int = 6, query_per_id: int = 1, gallery_per_id: int = 3,
                             size: Tuple[int, int] = (256, 128), max_id: int = 7999):
    """Factory for :class:`ReIDTaskPipeline`: deterministic ids per task name, disjoint across tasks."""
    def factory(task: str, split: str) -> ArrayReIDDataset:
        h = abs(hash_name(task))
        first = (h * num_ids) % max(1, (max_id + 1 - num_ids))
        ids = list(range(first, first + num_ids))
        per = {"train": train_per_id, "query": query_per_id, "gallery": gallery_per_id}[split]
        return make_array_split(ids, per, size, seed=h % 65521 + {"train": 0, "query": 1, "gallery": 2}[split])
    return factory


def hash_name(name: str) -> int:
    v = 2166136261
    for ch in name.encode():
        v = ((v ^ ch) * 16777619) & 0xFFFFFFFF
    return v


def write_imagefolder_tree(datasets_dir: str, tasks: Sequence[str], num_ids: int = 6, train_per_id: int = 4,
                           query_per_id: int = 1, gallery_per_id: int = 2, size: Tuple[int, int] = (128, 64),
                           max_id: int = 7999) -> Dict[str, Sequence[int]]:
    from PIL import Image
    out = {}
    fac = synthetic_source_factory(num_ids, train_per_id, query_per_id, gallery_per_id, size, max_id)
    for task in tasks:
        for split in ("train", "query", "gallery"):
            ds = fac(task, split)
            counters: Dict[int, int] = {}
            for i in range(len(ds)):
                img, pid, _ = ds[i]
                d = os.path.join(datasets_dir, task, split, str(pid))
                os.makedirs(d, exist_ok=True)
                k = counters.get(pid, 0)
                counters[pid] = k + 1
                Image.fromarray(img.numpy()).save(os.path.join(d, f"{k:04d}.jpg"), quality=95)
            out[task] = ds.person_ids
    return out


def clustered_features(num_query: int, num_gallery: int, dim: int, num_ids: int, seed: int = 0, spread: float = 0.6,
                       device="cpu"):
    """Seeded synthetic ReID embeddings: one random unit centre per identity, every image its identity's centre plus
    isotropic noise (``spread`` = noise norm relative to the centre), L2-normalised. Query and gallery identities are
    drawn independently and uniformly from ``num_ids``. Returns ``(query [Q, dim], q_labels, gallery [G, dim],
    g_labels)`` as fp32 / int64 tensors on ``device``. (Used by the re-ranking tests and ``scripts/rerank_bench.py``.)"""
    g = torch.Generator().manual_seed(seed)
    centres = torch.nn.functional.normalize(torch.randn(num_ids, dim, generator=g), dim=1)

    def draw(n):
        lab = torch.randint(0, num_ids, (n,), generator=g)
        x = centres[lab] + spread * torch.randn(n, dim, generator=g) / dim ** 0.5
        return torch.nn.functional.normalize(x, dim=1).to(device), lab.to(device)
    q, ql = draw(num_query)
    gf, gl = draw(num_gallery)
    return q, ql, gf, gl

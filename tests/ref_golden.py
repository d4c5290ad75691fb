"""Runs a whole (tiny) experiment of the UNMODIFIED reference in oracle/_ref as a golden oracle.

    python tests/ref_golden.py <in.pt> <out.pt>

``in.pt``: ``{"common": ..., "exp": ..., "rounds": R, "splits": {(task, split): (uint8 [N,H,W,3], pids [N])}}``.
``out.pt``: ``{"init": {role: plain net state_dict at construction}, "files": {relative ckpt path: object},
"log": experiment-log dict}``. The reference is driven through ``builder.parser_server / parser_clients`` and
``ExperimentStage._process_one_round``; the accommodations are those of SURVEY §8 (no network, in-memory splits).
"""
import logging
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
sys.path.insert(0, ROOT)
from baseline.reference_arm import _MemoryPipeline  # noqa: E402  (duck-typed pipeline, no reference import inside)

sys.path.insert(0, REF)
logging.disable(logging.CRITICAL)


def main():
    inp, outp = sys.argv[1:3]
    d = torch.load(inp, weights_only=False)
    common, exp, rounds = d["common"], d["exp"], d["rounds"]

    import numpy as np
    import torchvision
    import models as ref_models
    import models.resnet as ref_resnet
    import tools.evaluate as ref_eval

    def _fake_url_loader(url, *a, **k):
        name = [k_ for k_, v in ref_resnet.model_urls.items() if v == url][0]
        return getattr(torchvision.models, name)(weights=None).state_dict()

    ref_resnet.load_state_dict_from_url = _fake_url_loader

    import models.swin_transformer as ref_swin
    _SWIN = {"swin_tiny": dict(embed_dim=96, depths=(2, 2, 6, 2), num_heads=(3, 6, 12, 24)),
             "swin_small": dict(embed_dim=96, depths=(2, 2, 18, 2), num_heads=(3, 6, 12, 24)),
             "swin_base": dict(embed_dim=128, depths=(2, 2, 18, 2), num_heads=(4, 8, 16, 32)),
             "swin_large": dict(embed_dim=192, depths=(2, 2, 18, 2), num_heads=(6, 12, 24, 48))}

    _swin_cache = {}

    def _fake_swin_loader(url, *a, **k):
        # ONE "pre-trained" file for every model, as in real use. (The reference never ships parameters owned by
        # non-leaf modules - Swin's relative_position_bias_table - from the server to its clients, fedstil.py:482-486;
        # with a shared pre-trained file that is invisible, with per-model random tables it would not be.)
        name = [k_ for k_, v in ref_swin.model_urls.items() if v == url][0]
        if name not in _swin_cache:
            _swin_cache[name] = ref_swin.SwinTransformer(patch_size=4, window_size=7, **_SWIN[name]).state_dict()
        return {"model": {k_: v.clone() for k_, v in _swin_cache[name].items()}}

    ref_swin.load_state_dict_from_url = _fake_swin_loader
    if exp["model_opts"].get("drop_path_rate") == 0.0:
        # determinism shim: the reference hard-codes drop_path_rate=0.1 (swin_transformer.py:640-662) and draws the
        # per-sample keep mask from the global RNG; stochastic depth is switched off on both sides
        ref_swin.DropPath.forward = lambda self, x: x
    # restore the pinned-stack behaviour of np.argwhere(tensor) (see tests/ref_oracle.py) so mAP is the intended one
    _aw = np.argwhere
    ref_eval.np.argwhere = lambda a: _aw(a.numpy() if isinstance(a, torch.Tensor) else a)

    captured = []
    name = exp["model_opts"]["name"]
    orig = ref_models.nets[name]

    def factory(**kw):
        net = orig(**kw)
        captured.append({k: v.detach().clone() for k, v in net.state_dict().items()})
        return net

    ref_models.nets[name] = factory

    from builder import parser_clients, parser_server
    from datasets.datasets_loader import ReIDImageDataset
    from experiment import ExperimentLog, ExperimentStage
    from tools.utils import same_seeds
    from torch.utils.data import DataLoader

    aug = exp["task_opts"]["augment_opts"]
    mean = torch.tensor(aug["norm_mean"]).view(3, 1, 1)
    std = torch.tensor(aug["norm_std"]).view(3, 1, 1)

    def make_split(task, split):
        u8, pids = d["splits"][(task, split)]
        classes = sorted(set(pids.tolist()))                 # ImageFolder: class index = rank of the directory name
        src = {}
        for i, pid in enumerate(pids.tolist()):
            img = ((u8[i].permute(2, 0, 1).float() / 255.0) - mean) / std
            src.setdefault(pid, []).append((img, classes.index(pid)))
        return src

    class _Split(ReIDImageDataset):
        """In-memory split that looks like the reference's ImageFolder branch: ``classes`` is the LIST of person ids
        (index = class index), which is what ``person_ids`` hands to ``fedstil.py:923,956`` / ``icarl.py``."""

        def reload_source(self, source, transform=None):
            self.dataset = []
            self.classes = sorted(source)
            for pid, items in source.items():
                for img, cidx in items:
                    self.dataset.append((img, cidx))

    os.makedirs(common["checkpoints_dir"], exist_ok=True)
    os.makedirs(common["logs_dir"], exist_ok=True)
    same_seeds(exp["random_seed"])
    server = parser_server(exp, common)
    clients = parser_clients(exp, common)
    init = {exp["server"]["server_name"]: captured[0]}
    for c, sd in zip(clients, captured[1:]):
        init[c.client_name] = sd
    if exp["exp_method"] == "icarl":       # its Model wrapper swaps in a freshly initialised n_classes-wide classifier
        snap = lambda m: {k: v.detach().clone() for k, v in m.net.state_dict().items()}  # noqa: E731
        init = {exp["server"]["server_name"]: snap(server.model), **{c.client_name: snap(c.model) for c in clients}}
    for c in clients:
        c.task_pipeline = _MemoryPipeline(c.task_pipeline.task_list, exp["task_opts"], make_split, DataLoader, _Split)
    stage = ExperimentStage(common, [exp])
    log = ExperimentLog(os.path.join(common["logs_dir"], "golden.json"))
    same_seeds(exp["random_seed"])
    if d.get("val0"):                      # the reference's initial validation pass (experiment.py:163-173), sequential
        for c in clients:
            stage._process_val(c, log, 0, stage.container)
    for r in range(1, rounds + 1):
        stage._process_one_round(r, server, clients, exp, log)

    files = {}
    root = os.path.join(common["checkpoints_dir"], exp["exp_name"])
    for dirpath, _, names in os.walk(root):
        for n in names:
            p = os.path.join(dirpath, n)
            files[os.path.relpath(p, root)] = torch.load(p, map_location="cpu", weights_only=False)
    torch.save({"init": init, "files": files, "log": log.records}, outp)


if __name__ == "__main__":
    main()

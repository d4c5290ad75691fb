"""Runs pieces of the UNMODIFIED reference (installed in oracle/_ref) as an oracle. Executed in a SUBPROCESS by
tests/test_reference_parity.py because the reference's top-level package names (datasets, models, tools, ...) must
not leak into the test process.   python tests/ref_oracle.py <case> <in.pt> <out.pt>"""
import logging
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
sys.path.insert(0, REF)
logging.disable(logging.CRITICAL)


class _Log:
    def info(self, *a, **k): pass
    warn = warning = error = debug = info


def main():
    case, inp, outp = sys.argv[1:4]
    d = torch.load(inp, weights_only=False)
    if case == "evaluate":
        import numpy as np
        import tools.evaluate as E
        raw_cmc, raw_map = E.evaluate(d["qf"], d["ql"], d["gf"], d["gl"], device="cpu")
        # On the reference's pinned stack (torch 1.11 / numpy 1.2x) ``np.argwhere(tensor)`` yields an ``[R, 1]`` numpy
        # array; on torch 2.x it yields a ``[1, R]`` tensor, so ``len(right_result_index)`` becomes 1 and the AP loop
        # only scores the FIRST hit. The shim restores the pinned-stack behaviour (the intended trapezoid AP).
        _aw = np.argwhere
        E.np.argwhere = lambda a: _aw(a.numpy() if isinstance(a, torch.Tensor) else a)
        cmc, mAP = E.evaluate(d["qf"], d["ql"], d["gf"], d["gl"], device="cpu")
        out = {"cmc": torch.as_tensor(cmc).float(), "mAP": float(mAP), "raw_cmc": torch.as_tensor(raw_cmc).float(),
               "raw_mAP": float(raw_map)}
        E.np.argwhere = _aw
    elif case == "distance":
        from tools.distance import compute_cosine_distance, compute_euclidean_distance, compute_kl_distance
        out = {"eu": compute_euclidean_distance(d["a"], d["b"]), "cos": compute_cosine_distance(d["a"], d["b"]),
               "kl": compute_kl_distance(d["a"][:1], d["b"][:1])}
    elif case == "losses":
        from criterions.cross_entropy import CrossEntropyLabelSmooth
        from criterions.triplet_loss import TripletLoss
        score = d["score"].clone().requires_grad_(True)
        ce = CrossEntropyLabelSmooth(num_classes=score.shape[1], epsilon=0.1)
        l1 = ce(score=score, feature=None, target=d["target"])
        l1.backward()
        feat = d["feat"].clone().requires_grad_(True)
        res = {"ce": l1.detach(), "ce_grad": score.grad}
        for name, kw in (("tri_hard", dict(margin=0.3, hard_mining=True)), ("tri_soft", dict(margin=0, hard_mining=True)),
                         ("tri_w", dict(margin=0.3, hard_mining=False, norm_feat=True))):
            t = TripletLoss(**kw)
            res[name] = t(score=None, feature=feat, target=d["target"]).detach()
        if "teacher" in d:                      # dead code in the reference (not registered), still its definition
            from criterions.kd_loss import DistillKL
            res["kd"] = DistillKL(temperature=d["T"])(d["score"], d["teacher"]).detach()
        out = res
    elif case == "fedavg_calculate":
        from methods.fedavg import Server
        srv = Server.__new__(Server)
        srv.clients = d["clients"]
        srv.logger = _Log()
        got = {}
        srv.update_model = lambda merged: got.update(merged)
        srv.calculate()
        out = got
    elif case == "fedstil_dispatch":
        from methods.fedstil import Server
        srv = Server.__new__(Server)
        srv.clients = d["clients"]
        srv.token_memory = d["token_memory"]
        srv.distance_calculate_step, srv.distance_calculate_decay = d["step"], d["decay"]
        srv.logger = _Log()
        out = {name: srv.get_dispatch_incremental_state(name)["incremental_shared_params"] for name in d["receivers"]}
    elif case == "fedcurv_penalty":
        import torch.nn as nn
        from methods.fedcurv import Model
        m = Model.__new__(Model)
        nn.Module.__init__(m)
        m.lambda_penalty = d["lam"]
        m.params = {n: p.clone().requires_grad_(True) for n, p in d["params"].items()}
        m.precision_matrices = d["F"]
        m.params_old = d["p_old"]
        m.other_precision_matrices = d["others"]            # [(F_j dict, p_j dict), ...]
        loss = m.penalty()
        loss.backward()
        out = {"value": loss.detach(), "grads": {n: p.grad for n, p in m.params.items()}}
    elif case == "importance":
        import torch.nn as nn
        import torch.nn.functional as F
        method = d["method"]
        mod = __import__(f"methods.{method}", fromlist=["Model"])
        net = nn.Sequential(nn.Linear(6, 5), nn.ReLU(), nn.Linear(5, 4))
        net.load_state_dict(d["state"])

        class _Op:
            def _invoke_train(self, model, data, target, **kw):
                return {"loss": F.cross_entropy(model(data), target)}

        m = mod.Model.__new__(mod.Model)
        nn.Module.__init__(m)
        m.net = net
        m.operator = _Op()
        m.params = {n: p for n, p in net.named_parameters() if p.requires_grad}
        m.recall_dataloaders = {name: [(x, y, y) for x, y in batches] for name, batches in d["loaders"].items()}
        out = {n: t.detach() for n, t in m._calculate_importance().items()}
    elif case == "fedstil_layer_steps":
        from methods.fedstil import AdaptiveLayer
        layer = AdaptiveLayer(global_weight=d["G"].clone(), atten_default=d["atten"])
        params = [p for p in layer.parameters() if p.requires_grad]
        opt = (torch.optim.Adam(params, lr=d["lr"], weight_decay=d["wd"]) if d["opt"] == "adam"
               else torch.optim.SGD(params, lr=d["lr"], weight_decay=d["wd"]))
        thetas = []
        for x, t in zip(d["xs"], d["ts"]):
            opt.zero_grad()
            loss = ((layer(x) - t) ** 2).mean()
            # the sparseness regulariser of fedstil.py:639-644
            loss = loss + d["lam1"] * (torch.norm(layer.initial_global_weight_atten - layer.global_weight_atten, p=1) +
                                       torch.norm(layer.initial_adaptive_weight - layer.adaptive_weight, p=1))
            loss.backward()
            opt.step()
            thetas.append((layer.global_weight_atten * layer.global_weight + layer.adaptive_weight).detach().clone())
        out = {"thetas": thetas}
    elif case == "swin_forward":
        from models.swin_transformer import SwinTransformer
        net = SwinTransformer(img_size=d["img"], embed_dim=d["dim"], depths=d["depths"], num_heads=d["heads"],
                              window_size=d["ws"], num_classes=d["classes"], drop_path_rate=0.0).eval()
        missing, unexpected = net.load_state_dict(d["state"], strict=False)     # this engine's weights, same keys
        with torch.no_grad():
            out = {"missing": list(missing), "unexpected": list(unexpected), "feat": net.forward_features(d["x"]),
                   "logits": net(d["x"])}
    elif case == "schedule":
        from datasets.datasets_pipeline import ReIDTaskPipeline
        out = {}
        for sustain in d["sustain"]:
            pipe = ReIDTaskPipeline(list(d["tasks"]), {"sustain_rounds": sustain}, "unused")
            pipe.get_task = lambda idx=-1: pipe.task_list[idx]            # no datasets on disk: report the task name
            seq = []
            for _ in range(d["calls"]):
                seq.append((pipe.next_task(), pipe.current_task_idx, list(pipe.task_round_rest), pipe.reach_final_task()))
            out[sustain] = seq
    elif case == "explog":
        from experiment import ExperimentLog
        log = ExperimentLog(d["path"])
        for key, value in d["ops"]:
            log.record(key, value)
        import json
        out = {"records": log.records, "file": json.load(open(d["path"]))}
    elif case == "logger":
        logging.disable(logging.NOTSET)
        from tools.logger import Logger
        msgs = []

        class _H(logging.Handler):
            def emit(self, record):
                msgs.append(record.getMessage())

        lg = Logger("client-0")
        lg.logger.addHandler(_H())
        lg.logger.propagate = False
        lg.info_train("task-0-1", "cuda:0", 12345, 0.98765, 1.23456, 3, 5)
        lg.info_train("task-0-1", "cpu", 7, 0.5, 0.25)
        lg.info_validation("task-0-1", 1234, 56789, d["cmc"], 0.4321)
        out = msgs
    elif case == "analyse":
        # the analysis modules import matplotlib at module level (not installed here): empty stand-ins, the table
        # functions under test never touch them
        import contextlib
        import io
        import types
        for name in ("matplotlib", "matplotlib.ticker", "matplotlib.pyplot"):
            sys.modules.setdefault(name, types.ModuleType(name))
        sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
        sys.modules["matplotlib"].ticker = sys.modules["matplotlib.ticker"]
        import analyse.accuracy as ra
        import analyse.forgetting as rf
        out = {}
        for rnd in d["rounds"]:
            buf = io.StringIO()
            with contextlib.redirect_stdout(buf):
                ra.accuracy_on_round(d["logs"], rnd, d["metric"], "metric")
                rf.forgetting_on_round(d["logs"], rnd, d["metric"], "metric")
            out[rnd] = buf.getvalue()
    else:
        raise SystemExit(f"unknown case {case}")
    torch.save(out, outp)


if __name__ == "__main__":
    main()

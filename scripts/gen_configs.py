"""Generates ``configs/``: ``common.yaml`` plus every experiment family of the reference (15 basis experiments,
9 backbone experiments, 22 FedSTIL hyper-parameter sweeps - same ``exp_name`` / ``exp_method`` / hyper-parameters, so
``python main.py --experiments configs/basis_exp/experiment_fedstil.yaml`` means the same run) and the B200 workloads
named in BASELINE.json (``configs/b200/``: ResNet-50 / Swin-T, 8 clients x 5 tasks, 256x128, bf16).
Synaptic Intelligence (``basis_exp/experiment_si.yaml``, ``b200/experiment_si_res50_1.yaml``) is this project's
addition next to the reference's EWC / MAS experiments.

The experiment definitions are parameter tables below; files are emitted in a compact flow style."""
import os
import sys

import yaml

ROOT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "configs")
FT_RES, FT_SWIN = ["base.layer4", "classifier"], ["base.layers.3", "classifier"]
SERVER = {"server_name": "server"}
STIL_SERVER = {"server_name": "server", "distance_calculate_step": 10, "distance_calculate_decay": 0.8}


def net(name="resnet18", ft=None, **extra):
    d = {"name": name, "num_classes": 8000, "last_stride": 1, "neck": "bnneck"}
    d.update(extra)
    d["fine_tuning"] = ft or (FT_SWIN if name.startswith("swin") else FT_RES)
    return d


def clients(n=5, tasks=6, ckpt=None):
    out = []
    for i in range(n):
        c = {"client_name": f"client-{i}"}
        if ckpt:
            c["model_ckpt_name"] = ckpt
        c["tasks"] = [f"task-{i}-{t}" for t in range(tasks)]
        out.append(c)
    return out


def stil(name, atten=0.9, l1=1e-4, k=18000, backbone="resnet18", method="fedstil"):
    return {"exp_name": name, "exp_method": method,
            "model_opts": net(backbone, atten_default=atten, lambda_l1=l1, lambda_k=k), "server": dict(STIL_SERVER),
            "clients": clients(ckpt="fedstil_model")}


def weit(name, backbone="resnet18", l2=1e-3):
    return {"exp_name": name, "exp_method": "fedweit",
            "model_opts": net(backbone, lambda_l1=5e-6, lambda_l2=l2, lambda_mask=0.0, kb_cnt=5),
            "server": dict(SERVER), "clients": clients()}


def curv(name, backbone="resnet18", lam=50.0):
    return {"exp_name": name, "exp_method": "fedcurv", "model_opts": net(backbone, lambda_penalty=lam),
            "server": dict(SERVER), "clients": clients()}


BASIS = {
    "sm": {"exp_name": "sm", "exp_method": "baseline", "server": dict(SERVER), "clients": clients(ckpt="sm-model")},
    "mm": {"exp_name": "mm", "exp_method": "baseline", "server": dict(SERVER), "clients": clients()},
    "ewc": {"exp_name": "ewc", "exp_method": "ewc", "model_opts": net(lambda_penalty=50.0), "server": dict(SERVER),
            "clients": clients()},
    "mas": {"exp_name": "mas", "exp_method": "mas", "model_opts": net(lambda_penalty=0.01), "server": dict(SERVER),
            "clients": clients()},
    "si": {"exp_name": "si", "exp_method": "si", "model_opts": net(lambda_penalty=0.1, si_xi=1e-3),
           "server": dict(SERVER), "clients": clients()},
    "icarl": {"exp_name": "icarl", "exp_method": "icarl", "server": dict(SERVER),
              "model_opts": dict(net(k=12000, n_classes=10, examplar_batch_size=64), num_classes=10),
              "clients": clients()},
    "fedavg": {"exp_name": "fedavg", "exp_method": "fedavg", "server": dict(SERVER), "clients": clients()},
    "fedprox": {"exp_name": "fedprox", "exp_method": "fedprox", "model_opts": net(lambda_l2=1e-5),
                "server": dict(SERVER), "clients": clients()},
    "fedcurv": curv("fedcurv"),
    "fedweit": weit("fedweit"),
    "fedstil": stil("fedstil"),
    "fedstil_atten": stil("fedstil-atten", atten=0.0, l1=1e-5, method="fedstil-atten"),
    "fedstil_wo_al": stil("fedstil-wo-al", atten=1.0),
    "fedstil_wo_pr": stil("fedstil-wo-pr", k=0),
    "fedstil_wo_pt": stil("fedstil-wo-pt", l1=0.0),
    "fedstil_wo_st": stil("fedstil-wo-st", atten=0.0),
}
BACKBONE = {
    "fedcurv_res18": curv("fedcurv-res18"), "fedcurv_res50": curv("fedcurv-res50", "resnet50", 10.0),
    "fedcurv_swin": curv("fedcurv-swin", "swin_transformer_tiny", 5.0),
    "fedstil_res18": stil("fedstil-res18", k=12000), "fedstil_res50": stil("fedstil-res50", l1=1e-3, k=12000,
                                                                           backbone="resnet50"),
    "fedstil_swin": stil("fedstil-swin", l1=1e-3, k=12000, backbone="swin_transformer_tiny"),
    "fedweit_res18": weit("fedweit-res18"), "fedweit_res50": weit("fedweit-res50", "resnet50"),
    "fedweit_swin": weit("fedweit-swin", "swin_transformer_tiny", 1e-5),
}
INIT = {**{f"fedstil_a_{i}": stil(f"fedstil_a_{i}", atten=round(i / 10, 1)) for i in range(11)},
        **{f"fedstil_k_{i}": stil(f"fedstil_k_{i}", k=2000 * i) for i in range(11)}}

COMMON = {
    "datasets_dir": "./datasets/preprocessed_shuffle/", "checkpoints_dir": "./ckpts/", "logs_dir": "./logs/",
    "parallel": 1, "device": ["cuda:0"],
    "defaults": {
        "random_seed": 123,
        "exp_opts": {"comm_rounds": 60, "val_interval": 10, "online_clients": 5},
        "model_opts": net(),
        "criterion_opts": {"name": "cross_entropy", "num_classes": 8000, "epsilon": 0.1},
        "optimizer_opts": {"name": "adam", "lr": 1.0e-3, "weight_decay": 1.0e-5},
        "scheduler_opts": {"name": "step_lr", "step_size": 5},
        "task_opts": {"sustain_rounds": 10, "train_epochs": 5,
                      "augment_opts": {"level": "default", "img_size": [128, 64], "norm_mean": [0.485, 0.456, 0.406],
                                       "norm_std": [0.229, 0.224, 0.225]},
                      "loader_opts": {"batch_size": 64, "num_workers": 0, "pin_memory": False,
                                      "persistent_workers": False, "multiprocessing_context": None}},
        "engine_opts": {"compute_dtype": "bf16", "async_checkpoint": True, "save_payload_ckpts": True,
                        "device_augment": True, "reference_compat": True},
    },
}


def b200(name, method, backbone, **model_extra):
    exp = {"exp_name": name, "exp_method": method,
           "exp_opts": {"comm_rounds": 50, "val_interval": 10, "online_clients": 8},
           "model_opts": net(backbone, **model_extra),
           "task_opts": dict(COMMON["defaults"]["task_opts"], train_epochs=1,
                             augment_opts=dict(COMMON["defaults"]["task_opts"]["augment_opts"], img_size=[256, 128])),
           "server": dict(STIL_SERVER if method.startswith("fedstil") else SERVER),
           "clients": clients(8, 5, "fedstil_model" if method.startswith("fedstil") else None)}
    return exp


B200 = {
    "fedstil_res50_8x5": b200("b200-fedstil-res50", "fedstil", "resnet50", atten_default=0.9, lambda_l1=1e-3,
                              lambda_k=12000),
    "fedstil_swin_8x5": b200("b200-fedstil-swin", "fedstil", "swin_transformer_tiny", atten_default=0.9,
                             lambda_l1=1e-3, lambda_k=12000),
    "fedcurv_res50_8": b200("b200-fedcurv-res50", "fedcurv", "resnet50", lambda_penalty=10.0),
    "fedavg_res50_2": dict(b200("b200-fedavg-res50-2c", "fedavg", "resnet50"), clients=clients(2, 1),
                           exp_opts={"comm_rounds": 5, "val_interval": 5, "online_clients": 2}),
    "ewc_res50_1": dict(b200("b200-ewc-res50", "ewc", "resnet50", lambda_penalty=50.0), clients=clients(1, 5),
                        exp_opts={"comm_rounds": 50, "val_interval": 10, "online_clients": 1}),
    "mas_res50_1": dict(b200("b200-mas-res50", "mas", "resnet50", lambda_penalty=0.01), clients=clients(1, 5),
                        exp_opts={"comm_rounds": 50, "val_interval": 10, "online_clients": 1}),
    "si_res50_1": dict(b200("b200-si-res50", "si", "resnet50", lambda_penalty=0.1, si_xi=1e-3), clients=clients(1, 5),
                       exp_opts={"comm_rounds": 50, "val_interval": 10, "online_clients": 1}),
    "icarl_res50_1": dict(b200("b200-icarl-res50", "icarl", "resnet50", k=12000, n_classes=10), clients=clients(1, 5),
                          exp_opts={"comm_rounds": 50, "val_interval": 10, "online_clients": 1}),
}


class _Flow(yaml.SafeDumper):
    pass


def _repr_list(dumper, data):
    flow = all(not isinstance(x, (dict, list)) for x in data)
    return dumper.represent_sequence("tag:yaml.org,2002:seq", data, flow_style=flow)


def _repr_dict(dumper, data):
    """Option groups whose values are scalars (or short scalar lists) are written on one line."""
    leaf = bool(data) and all(not isinstance(v, dict) and not (isinstance(v, list) and any(isinstance(x, (dict, list)) for x in v))
                             for v in data.values())
    return dumper.represent_mapping("tag:yaml.org,2002:map", data, flow_style=leaf and len(data) <= 8)


_Flow.add_representer(list, _repr_list)
_Flow.add_representer(dict, _repr_dict)


def emit(path, obj, header):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        f.write(f"# {header}\n# generated by scripts/gen_configs.py - edit the tables there\n")
        yaml.dump(obj, f, Dumper=_Flow, sort_keys=False, width=110)


def main():
    emit(os.path.join(ROOT, "common.yaml"), COMMON, "paths, devices and the defaults shallow-merged under every experiment")
    for fam, table in (("basis_exp", BASIS), ("backbone", BACKBONE), ("init_exp", INIT), ("b200", B200)):
        for key, exp in table.items():
            emit(os.path.join(ROOT, fam, f"experiment_{key}.yaml"), exp, f"{fam}: {exp['exp_name']} ({exp['exp_method']})")
    print("wrote", sum(len(t) for t in (BASIS, BACKBONE, INIT, B200)) + 1, "files under", ROOT)


if __name__ == "__main__":
    main()

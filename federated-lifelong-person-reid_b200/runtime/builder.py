"""Object construction from configuration (``builder.py:16-104``): ``parser_model / parser_criterion /
parser_optimizer / parser_scheduler / parser_server / parser_clients``.

Semantics kept: freeze everything then un-freeze the ``fine_tuning`` sub-modules by name; wrap in the method's
``Model`` when it defines one; ``model_opts`` minus ``name/fine_tuning`` goes to **both** the net constructor and the
method ``Model`` constructor; the optimizer only sees ``requires_grad`` parameters; extra ``server:`` / ``clients[i]:``
keys become constructor kwargs.

Differences: models are materialised on their device at build time (flat arena, bf16 shadow, tensor-core head), and
only the clients *hosted on this rank* are instantiated (``client_id % world_size == rank``).
"""
from __future__ import annotations

import os
from typing import Any, Callable, Dict, List, Optional

import torch
import torch.nn as nn

from ..criterions import criterions
from ..data.pipeline import ReIDTaskPipeline
from ..methods import methods
from ..models import nets, optimizers, schedulers
from ..ops.rank import re_ranking_params
from .checkpoint import CheckpointStore
from .modules import ClientModule, ModelModule, ServerModule


_INIT_CACHE: Dict[str, Dict] = {}


def _initial_state(engine_opts: Dict, role: Optional[str]) -> Optional[Dict[str, torch.Tensor]]:
    """``engine_opts.init_state``: path of a ``torch.save``d ``{role name: plain net state_dict}`` table (role = server
    or client name; ``"*"`` = everyone) loaded into the freshly constructed net – the offline stand-in for the
    reference's ImageNet download (``models/resnet.py:308-310``) and the hook the golden-parity tests use."""
    path = engine_opts.get("init_state")
    if not path or role is None:
        return None
    if path not in _INIT_CACHE:
        _INIT_CACHE.clear()
        _INIT_CACHE[path] = torch.load(path, map_location="cpu", weights_only=False)
    table = _INIT_CACHE[path]
    return table.get(role, table.get("*"))


def _load_matching(net: nn.Module, state: Dict[str, torch.Tensor]) -> None:
    own = net.state_dict()
    with torch.no_grad():
        for k, v in state.items():
            if k in own and own[k].shape == v.shape:
                own[k].copy_(v)


def parser_model(method_name: str, model_config: Dict, device: str | torch.device = "cpu",
                 engine_opts: Optional[Dict] = None, role: Optional[str] = None) -> ModelModule:
    engine_opts = engine_opts or {}
    factory_kwargs = {n: p for n, p in model_config.items() if n not in ["name", "fine_tuning"]}
    if method_name == "fedstil-atten" and "num_clients" in engine_opts:
        factory_kwargs.setdefault("num_clients", engine_opts["num_clients"])
    net = nets[model_config["name"]](**factory_kwargs)
    init = _initial_state(engine_opts, role)
    if init is not None:
        _load_matching(net, init)
    if model_config.get("fine_tuning"):
        for p in net.parameters():
            p.requires_grad = False
        for layer_name in model_config["fine_tuning"]:
            for p in net.get_submodule(layer_name).parameters():
                p.requires_grad = True
        # the reference builds the BNNeck bias frozen and the blanket un-freeze does not touch it unless listed
    module = methods[method_name]
    model = module.Model(net=net, **factory_kwargs) if hasattr(module, "Model") else ModelModule(net)
    if init is not None:
        _load_matching(model.net, init)          # layers the method wrapper re-created (iCaRL's classifier)
    model.materialize(device, engine_opts.get("compute_dtype", "bf16"), model_config.get("fine_tuning"))
    return model


def parser_criterion(criterion_configs: Any) -> List[Callable]:
    if isinstance(criterion_configs, dict):
        criterion_configs = [criterion_configs]
    out = []
    for cfg in criterion_configs:
        kwargs = {n: p for n, p in cfg.items() if n != "name"}
        out.append(criterions[cfg["name"]](**kwargs))
    return out


def parser_optimizer(model: ModelModule, optim_config: Dict):
    kwargs = {n: p for n, p in optim_config.items() if n != "name"}
    return optimizers[optim_config["name"]](model.arena, **kwargs)


def parser_scheduler(optim, scheduler_config: Dict):
    kwargs = {n: p for n, p in scheduler_config.items() if n != "name"}
    return schedulers[scheduler_config["name"]](optimizer=optim, **kwargs)


def _operator(exp_config: Dict, model: ModelModule):
    criterion = parser_criterion(exp_config["criterion_opts"])
    for c in criterion:
        if isinstance(c, nn.Module):
            c.to(model.device)
    optimizer = parser_optimizer(model, exp_config["optimizer_opts"])
    scheduler = parser_scheduler(optimizer, exp_config["scheduler_opts"])
    return methods[exp_config["exp_method"]].Operator(method_name=exp_config["exp_method"], criterion=criterion,
                                                      optimizer=optimizer, scheduler=scheduler)


def parser_server(exp_config: Dict, common_config: Dict, device="cpu", store: Optional[CheckpointStore] = None,
                  comm=None) -> ServerModule:
    method = exp_config["exp_method"]
    for key in ("server_opt", "aggregator"):
        if key in exp_config["server"]:
            from ..methods.fedbase import FedServer
            if not issubclass(methods[method].Server, FedServer):
                # every other server role has its own aggregation (or none): the key would otherwise be dropped silently
                raise ValueError(f"server.{key} is only supported by fedavg, fedprox and fedcurv, not by {method!r}")
    eng = dict(exp_config.get("engine_opts", {}), num_clients=len(exp_config["clients"]))
    model = parser_model(exp_config["exp_method"], exp_config["model_opts"], device, eng,
                         exp_config["server"]["server_name"])
    operator = _operator(exp_config, model)
    kwargs = {n: p for n, p in exp_config["server"].items() if n != "server_name"}
    return methods[exp_config["exp_method"]].Server(
        server_name=exp_config["server"]["server_name"], model=model, operator=operator,
        ckpt_root=os.path.join(common_config["checkpoints_dir"], exp_config["exp_name"]), store=store, comm=comm,
        **kwargs)


def parser_clients(exp_config: Dict, common_config: Dict, device="cpu", store: Optional[CheckpointStore] = None,
                   comm=None, rank: int = 0, world: int = 1, source_factory=None) -> List[ClientModule]:
    """Instantiate the clients hosted on this rank (all of them when ``world == 1``)."""
    eng = dict(exp_config.get("engine_opts", {}), num_clients=len(exp_config["clients"]))
    clients = []
    for cid, client_config in enumerate(exp_config["clients"]):
        if cid % world != rank:
            continue
        model = parser_model(exp_config["exp_method"], exp_config["model_opts"], device, eng,
                             client_config["client_name"])
        operator = _operator(exp_config, model)
        pipeline = ReIDTaskPipeline(task_list=client_config["tasks"], task_opts=exp_config["task_opts"],
                                    datasets_dir=common_config["datasets_dir"],
                                    device_loader=eng.get("device_augment", True), source_factory=source_factory)
        kwargs = {n: p for n, p in client_config.items() if n not in ("client_name",)}
        kwargs.setdefault("reference_compat", eng.get("reference_compat", True))
        kwargs.setdefault("re_ranking", re_ranking_params(eng.get("re_ranking", False)))
        anchor = eng.get("train_l1_anchor")
        kwargs.setdefault("train_l1_anchor", bool(eng.get("reference_compat", True) if anchor is None else anchor))
        clients.append(methods[exp_config["exp_method"]].Client(
            client_name=client_config["client_name"], model=model, operator=operator,
            ckpt_root=os.path.join(common_config["checkpoints_dir"], exp_config["exp_name"]),
            task_pipeline=pipeline, store=store, client_id=cid, comm=comm, **kwargs))
    return clients

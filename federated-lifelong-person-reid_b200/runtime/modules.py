"""Abstract building blocks of a method plug-in: ``ModelModule``, ``OperatorModule``, ``ClientModule``,
``ServerModule`` (contracts of ``modules/{model,operator,client,server}.py`` in the reference).

What is kept: the public protocol (``get_incremental_state`` / ``set_client_incremental_state`` / ``calculate`` /
``get_dispatch_*_state`` / ``update_by_*_state`` / ``train`` / ``validate`` / ``inference``), the checkpoint helpers
and their on-disk layout, the ``**kwargs -> setattr`` convention.

What is different: models live on their device for the whole experiment (no ``model_on_device`` shuttle, no
load/save round-trip through disk around every call), the trainable state is a flat :class:`ParamArena`, and the
server is a *role* replicated on every rank whose aggregation runs as collectives of :class:`FedComm`.
"""
from __future__ import annotations

import contextlib
from typing import Any, Dict, List, Optional, Sequence, Tuple, Union

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..evaluation import evaluate
from ..utils.logger import Logger
from ..utils.trace import host_list
from .arena import ArenaOptimizer, ParamArena, StepLR
from .checkpoint import CheckpointStore


_RNG_STREAMS = 0


def _cuda(device) -> bool:
    return torch.device(device).type == "cuda"


class ModelModule(nn.Module):
    """Wraps a backbone ``net``; owns the trainable-parameter arena once :meth:`materialize` has been called."""

    def __init__(self, net: nn.Module, **kwargs):
        super().__init__()
        self.net = net
        self.args = kwargs
        self.arena: Optional[ParamArena] = None
        self.compute_dtype = torch.float32
        self.rng: Optional[torch.Generator] = None       # per-model device generator (see materialize)

    def forward(self, *args, **kwargs):
        return self.net(*args, **kwargs)

    def train(self, mode: bool = True):
        """``nn.Module.train`` walks ~160 sub-modules; the round loop toggles train / eval several times per client and
        round, mostly to the mode the model is already in."""
        if self.training == mode and getattr(self, "_mode_uniform", None) == mode:
            return self
        super().train(mode)
        self._mode_uniform = mode
        return self

    @property
    def device(self) -> torch.device:
        return next(self.parameters()).device

    # ---- arena ---------------------------------------------------------------------------------------------
    def upload_filter(self, name: str) -> bool:
        """Which trainable parameters form the upload prefix of the arena (default: all of them)."""
        return True

    def trainable_named_parameters(self) -> List[Tuple[str, nn.Parameter]]:
        return [(n, p) for n, p in self.net.named_parameters() if p.requires_grad]

    def materialize(self, device: Union[str, torch.device], compute_dtype: str = "bf16",
                    fine_tuning: Optional[Sequence[str]] = None) -> "ModelModule":
        """Move to ``device``, flatten the trainable parameters into an arena, enable the tensor-core head."""
        device = torch.device(device)
        self.to(device)
        self.compute_dtype = torch.bfloat16 if (device.type == "cuda" and compute_dtype == "bf16") else torch.float32
        if hasattr(self.net, "configure_split"):
            self.net.configure_split(fine_tuning)
        self.arena = ParamArena(self.trainable_named_parameters(), device,
                                shadow=self.compute_dtype == torch.bfloat16, first=self.upload_filter)
        if device.type == "cuda":
            # A private generator per model: sample shuffling / augmentation of one client never touch the default
            # CUDA generator, which another client's thread may have registered with an ongoing graph capture, and
            # a client's random stream does not depend on how the client threads interleave.
            global _RNG_STREAMS
            _RNG_STREAMS += 1
            self.rng = torch.Generator(device=device)
            self.rng.manual_seed((torch.initial_seed() + 7919 * _RNG_STREAMS) % (1 << 62))
        if device.type == "cuda" and self.compute_dtype == torch.bfloat16:
            from ..models.resnet import FastResNetHead, NativeTrunk, ResNetReID
            if isinstance(self.net, ResNetReID) and 1 <= self.net.head_start <= 4:
                self.net._fast_head = FastResNetHead(self.net, self.arena.shadow_of, self.arena.grad_of)
                if getattr(self, "use_native_trunk", True):
                    self.net._native_trunk = NativeTrunk(self.net)
            from ..models.swin import SwinTransformerReID, use_tensor_core_linears
            if isinstance(self.net, SwinTransformerReID) and getattr(self, "use_tc_linears", True):
                # every Linear of the backbone (qkv / proj / fc1 / fc2 / patch merging) and the classifier on the
                # wgmma GEMM: trainable ones with the optimizer-maintained bf16 copy and direct gradient slots
                use_tensor_core_linears(self.net, self.arena.shadow_of, self.arena.grad_of)
                from ..ops import layer as lops
                lops.enabled("swin_tokens", device)    # one-time on-device self-check of the token kernels, up front
        return self

    def autocast(self):
        if self.compute_dtype == torch.bfloat16:
            return torch.autocast(device_type="cuda", dtype=torch.bfloat16)
        return contextlib.nullcontext()

    def prepare_input(self, data: torch.Tensor) -> torch.Tensor:
        data = data.to(self.device, non_blocking=True)
        if data.dim() == 4 and self.device.type == "cuda":
            data = data.contiguous(memory_format=torch.channels_last)
        return data

    # ---- state dict helpers (contiguous copies; arena views are strided) --------------------------------------
    def full_state(self) -> Dict[str, torch.Tensor]:
        return {k: v.detach().clone(memory_format=torch.contiguous_format) for k, v in self.state_dict().items()}

    def load_full_state(self, state: Dict[str, torch.Tensor]) -> None:
        own = self.state_dict()
        with torch.no_grad():
            for k, v in state.items():
                if k in own:
                    own[k].copy_(v.to(own[k].device))
        if self.arena is not None:
            self.arena.refresh_shadow()

    def model_state(self, *args, **kwargs) -> Dict:
        return self.full_state()

    def update_model(self, params_state: Dict[str, torch.Tensor]) -> None:
        self.load_full_state(params_state)

    # ---- resume manifest (runtime/resume.py): method-specific continual-learning state -----------------------------
    resume_attrs: Tuple[str, ...] = ()       # names of tensor / scalar attributes that a continued run needs

    def resume_extra(self) -> Dict[str, Any]:
        out = {}
        for name in self.resume_attrs:
            v = getattr(self, name, None)
            out[name] = v.detach().clone() if isinstance(v, torch.Tensor) else v
        return out

    def load_resume_extra(self, extra: Dict[str, Any]) -> None:
        for name in self.resume_attrs:
            if name not in extra:
                continue
            v, cur = extra[name], getattr(self, name, None)
            if isinstance(v, torch.Tensor) and isinstance(cur, torch.Tensor) and cur.shape == v.shape:
                cur.copy_(v.to(cur.device))
            elif isinstance(v, torch.Tensor):
                setattr(self, name, v.to(self.device))
            else:
                setattr(self, name, v)


class OperatorModule:
    """Holds criterion list / optimizer / scheduler and the train / predict / valid / inference loops
    (``modules/operator.py`` + the canonical loops of ``methods/baseline.py:26-210``)."""

    def __init__(self, optimizer: ArenaOptimizer = None, criterion: List = None, scheduler: StepLR = None,
                 logger: Logger = None, **kwargs):
        self.logger = logger if logger is not None else Logger()
        self.criterion = criterion or []
        self.optimizer = optimizer
        self.scheduler = scheduler
        self.args = kwargs

    @staticmethod
    def iter_dataloader(*dataloaders):
        if len(dataloaders) == 1 and isinstance(dataloaders[0], list):
            dataloaders = dataloaders[0]
        for dl in dataloaders:
            for value in dl:
                yield value

    # ---- hooks --------------------------------------------------------------------------------------------------
    def compute_loss(self, model: ModelModule, score, feature, target) -> torch.Tensor:
        loss = 0.0
        for fn in self.criterion:
            loss = loss + fn(score=score, feature=feature, target=target)
        return loss

    def extra_loss_value(self, model: ModelModule, batches: int) -> float:
        """Penalty / regulariser value folded into the optimizer kernel, averaged per batch for reporting."""
        return 0.0

    def forward_train(self, model: ModelModule, data: torch.Tensor):
        with model.autocast():
            return model.forward(data)

    # Reference quirk (reference_compat): the Operators of fedstil / fedstil-atten / fedweit / icarl rebuild
    # ``optimizer.param_groups`` from ``optimizer.defaults`` at the top of every ``invoke_train``
    # (``set_optimizer_parameters``, e.g. fedstil.py:553-556,631), so whatever StepLR did to the lr is undone before
    # the next epoch - those methods always step with the configured lr. Their clients set this flag.
    reset_lr_each_epoch = False

    def begin_epoch(self) -> None:
        if self.reset_lr_each_epoch and self.optimizer is not None:
            self.optimizer.restore_default_lr()

    # ---- loops --------------------------------------------------------------------------------------------------
    def _invoke_train(self, model: ModelModule, data, target, **kwargs) -> Dict:
        score, feature = self.forward_train(model, data)
        return {"score": score, "feature": feature, "loss": self.compute_loss(model, score, feature, target)}

    # ---- CUDA-graph capture of one training step ------------------------------------------------------------------
    # A step of the ResNet path is ~400 kernel launches (native trunk + head forward / backward + fused optimizer)
    # whose Python dispatch costs several times their device time; the step is free of host synchronisation (loss /
    # accuracy accumulate on the device), so it is captured once per input shape and replayed.
    graph_step = True                  # sub-classes whose step is not capturable (host-side control flow) clear it

    def _ce_stats_ok(self, model: ModelModule) -> bool:
        """The fused CE kernel already produces the loss sum and the top-1 hit count on the device: when the only
        criterion is the label-smoothing CE over the classifier's full width, use its accumulator instead of a
        separate argmax / compare / sum chain (5 small kernels per step)."""
        from ..criterions import CrossEntropyLabelSmooth
        cls = getattr(model.net, "classifier", None)
        return (len(self.criterion) == 1 and isinstance(self.criterion[0], CrossEntropyLabelSmooth)
                and cls is not None and getattr(cls, "out_features", -1) == self.criterion[0].num_classes
                and model.device.type == "cuda")

    def _graph_capable(self, model: ModelModule) -> bool:
        return (self.graph_step and model.device.type == "cuda" and getattr(model, "use_cuda_graphs", True)
                and getattr(model.net, "thread_safe_rng", False) and getattr(model.net, "_fast_head", None) is not None)

    def _graphed_step(self, model: ModelModule):
        """One training step (zero-grad, forward, loss, backward, fused optimizer) as a replayable CUDA graph
        (eager on the CPU / when capture is not possible); loss / hit accumulators live in ``self._acc``."""
        st = getattr(self, "_step", None)
        if st is None:
            from .graphs import GraphedStep
            self._acc = torch.zeros(2, dtype=torch.float64, device=model.device)
            self._ce_acc = torch.zeros(2, dtype=torch.float32, device=model.device) if self._ce_stats_ok(model) \
                else None
            if self._ce_acc is not None:
                self.criterion[0].stats = self._ce_acc

            def fn(data, target):
                self.optimizer.zero_grad()
                out = self._invoke_train(model, data, target)
                out["loss"].backward()
                self.optimizer.step()
                if self._ce_acc is None:
                    with torch.no_grad():
                        self._acc[0] += out["loss"].detach().double()
                        self._acc[1] += (out["score"].argmax(dim=1) == target).sum()

            st = self._step = GraphedStep(fn, warmup=2, enabled=self._graph_capable(model))
        return st

    def _step_totals(self) -> Tuple[float, float]:
        """(loss sum, top-1 hits) accumulated by the steps since the accumulators were last zeroed: ONE host sync."""
        src = self._acc if self._ce_acc is None else self._ce_acc.double()
        loss_sum, hits = host_list(src)
        return loss_sum, hits

    def _zero_step_totals(self) -> None:
        self._acc.zero_()
        if self._ce_acc is not None:
            self._ce_acc.zero_()

    @staticmethod
    def _bn_counters(model: ModelModule, on: bool, add: int = 0) -> None:
        """``num_batches_tracked`` bookkeeping of the native trunk / head: one tiny kernel per BN layer per step ->
        one per BN layer per epoch."""
        for name in ("_native_trunk", "_fast_head"):
            fast = getattr(model.net, name, None)
            if fast is not None and model.device.type == "cuda":
                if add:
                    fast.add_batches(add)
                fast.count_batches = on

    def invoke_train(self, model: ModelModule, dataloader, **kwargs) -> Dict:
        device = model.device
        model.train()
        self.begin_epoch()
        batch_cnt = data_cnt = 0
        if self.optimizer.stats is not None:
            self.optimizer.stats.zero_()
        step = self._graphed_step(model)
        self._zero_step_totals()
        self._bn_counters(model, on=False)
        for data, person_id, classes_id in dataloader:
            data, target = model.prepare_input(data), person_id.to(device, non_blocking=True)
            step(data, target)
            data_cnt += len(data)
            batch_cnt += 1
        self._bn_counters(model, on=True, add=batch_cnt)
        loss_sum, hits = self._step_totals()                            # the only host sync of the epoch
        train_loss = loss_sum / max(batch_cnt, 1) + self.extra_loss_value(model, batch_cnt)
        if self.scheduler:
            self.scheduler.step()
        return {"accuracy": hits / max(data_cnt, 1), "loss": train_loss, "batch_count": batch_cnt,
                "data_count": data_cnt}

    def invoke_predict(self, model: ModelModule, dataloader, **kwargs) -> Dict:
        """No-grad evaluation in *train* mode (exists in every reference Operator, never called by its runtime)."""
        device = model.device
        model.train()
        acc = torch.zeros(2, dtype=torch.float64, device=device)
        batch_cnt = data_cnt = 0
        for data, person_id, classes_id in dataloader:
            data, target = model.prepare_input(data), person_id.to(device)
            with torch.no_grad():
                out = self._invoke_train(model, data, target, **kwargs)
                acc[0] += out["loss"].double()
                acc[1] += (out["score"].argmax(dim=1) == target).sum()
            data_cnt += len(data)
            batch_cnt += 1
        loss_sum, hits = host_list(acc)
        return {"accuracy": hits / max(data_cnt, 1), "loss": loss_sum / max(batch_cnt, 1), "batch_count": batch_cnt,
                "data_count": data_cnt}

    def _invoke_valid(self, model: ModelModule, data, target=None, norm: bool = True, **kwargs) -> Dict:
        with model.autocast():
            feat = model.forward(data)
        feat = feat.float()
        if norm:
            feat = F.normalize(feat, dim=1, p=2)
        return {"feature": feat}

    _invoke_inference = _invoke_valid

    def invoke_valid(self, model: ModelModule, dataloader, **kwargs) -> Dict:
        """Features stay on the device (the reference ships them to the host and back, baseline.py:189-190)."""
        batch_cnt = data_cnt = 0
        features, labels = [], []
        model.eval()
        for data, person_id, classes_id in dataloader:
            data = model.prepare_input(data)
            with torch.no_grad():
                features.append(self._invoke_valid(model, data, None)["feature"])
                labels.append(person_id.to(model.device))
            batch_cnt += 1
            data_cnt += len(data)
        if features:
            features, labels = torch.cat(features, 0), torch.cat(labels, 0)
        else:
            features, labels = torch.zeros(0, 1, device=model.device), torch.zeros(0, dtype=torch.long)
        return {"features": features, "labels": labels, "batch_count": batch_cnt, "data_count": data_cnt}

    def invoke_inference(self, model: ModelModule, dataloader, **kwargs) -> Dict:
        out = self.invoke_valid(model, dataloader, **kwargs)
        out.pop("labels", None)
        return out


class _Actor:
    """Checkpoint helpers shared by clients and servers (``{ckpt_root}/{actor}/{state}.ckpt``)."""

    name: str
    store: CheckpointStore

    def load_state(self, state_name: str, default_value: Any = None) -> Any:
        return self.store.load(self.name, state_name, default_value)

    def save_state(self, state_name: Optional[str], state: Any, cover: bool = False) -> None:
        self.store.save(self.name, state_name, state, cover)

    def load_model(self, model_name: str) -> None:
        """Explicit restore from disk (resume). The engine never needs it between rounds: state is resident."""
        if self.store.exists(self.name, model_name):
            self.model.update_model(self.load_state(model_name))

    def save_model(self, model_name: str) -> None:
        self.save_state(model_name, self.model.model_state(), True)

    def update_model(self, params_state: Dict[str, torch.Tensor]) -> None:
        self.model.update_model(params_state)


class ClientModule(_Actor):
    def __init__(self, client_name: str, model: ModelModule, operator: OperatorModule, ckpt_root: str,
                 model_ckpt_name: str = None, store: Optional[CheckpointStore] = None, client_id: int = 0,
                 comm=None, **kwargs):
        self.client_name = self.name = client_name
        self.client_id = client_id
        self.model = model
        self.operator = operator
        self.comm = comm
        for n, p in kwargs.items():
            setattr(self, n, p)
        self.store = store if store is not None else CheckpointStore(ckpt_root, asynchronous=False)
        self.ckpt_path = self.store.path(client_name, "")[:-5].rstrip("/")
        self.model_ckpt_name = model_ckpt_name
        self.logger = Logger(f"{client_name}")
        self.operator.logger = self.logger
        self.train_cnt = 0
        self.test_cnt = 0
        self.logger.info("Startup successfully.")

    # ---- protocol stubs (modules/client.py:78-88) ---------------------------------------------------------------
    def get_incremental_state(self, **kwargs) -> Optional[Dict]:
        return None

    def get_integrated_state(self, **kwargs) -> Optional[Dict]:
        return None

    def update_by_incremental_state(self, state: Dict, **kwargs) -> Any:
        return None

    def update_by_integrated_state(self, state: Dict, **kwargs) -> Any:
        return None

    # ---- shared train / validate skeleton -----------------------------------------------------------------------
    def ckpt_name(self, task_name: str) -> str:
        return self.model_ckpt_name if self.model_ckpt_name else task_name

    def train_one_epoch(self, task_name: str, tr_loader, val_loader, **kwargs) -> Dict:
        return self.operator.invoke_train(self.model, tr_loader)

    def before_train(self, task_name: str, tr_loader, val_loader) -> None:
        pass

    def after_epoch(self, output: Dict) -> None:
        pass

    def after_train(self, task_name: str, tr_loader, val_loader, output: Dict) -> None:
        pass

    def train(self, epochs: int, task_name: str, tr_loader, val_loader, early_stop_threshold: int = 3,
              device: str = "cpu", **kwargs) -> Dict:
        """Epoch loop with the reference's early stopping (``methods/baseline.py:227-268``)."""
        _bind_loader(tr_loader, self.model)
        self.before_train(task_name, tr_loader, val_loader)
        output: Dict = {}
        perf_loss, perf_acc, sustained = 1e8, 0, 0
        from ..utils.trace import nvtx_range
        for epoch in range(1, epochs + 1):
            with nvtx_range(f"{self.client_name}/epoch{epoch}"):
                output = self.train_one_epoch(task_name, tr_loader, val_loader)
            accuracy, loss, data_count = output["accuracy"], output["loss"], output["data_count"]
            sustained += 1
            if loss <= perf_loss and accuracy >= perf_acc:
                perf_loss, perf_acc, sustained = loss, accuracy, 0
            if early_stop_threshold and sustained >= early_stop_threshold:
                break
            self.after_epoch(output)
            self.logger.info_train(task_name, self.model.device, data_count, perf_acc, perf_loss, epoch, epochs)
        self.after_train(task_name, tr_loader, val_loader, output)
        self.operator.optimizer.reset_state()
        with nvtx_range(f"{self.client_name}/checkpoint"):
            self.save_model(self.ckpt_name(task_name))
        return output

    def _features(self, loader) -> Dict:
        _bind_loader(loader, self.model)
        return self.operator.invoke_valid(self.model, loader)

    def validate(self, task_name: str, query_loader, gallery_loader, device: str = "cpu", **kwargs):
        gallery = self._features(gallery_loader)
        query = self._features(query_loader)
        self.test_cnt += len(gallery["features"]) + len(query["features"])
        # ``_ranker``: set by the experiment loop for ``engine_opts.sharded_validation`` (collective, gallery-sharded)
        rank_fn = getattr(self, "_ranker", None) or evaluate
        cmc, mAP = rank_fn(query["features"], query["labels"], gallery["features"], gallery["labels"])
        allf = torch.cat([query["features"], gallery["features"]], dim=0)
        avg_rep = allf.sum(dim=0) / max(len(allf), 1)
        self.logger.info_validation(task_name, len(query["features"]), len(gallery["features"]), cmc, mAP)
        rr = getattr(self, "re_ranking", None)
        if not rr:
            return cmc, mAP, avg_rep
        # ``engine_opts.re_ranking``: the same features ranked again by the k-reciprocal distance (ops/rank.py)
        rr_cmc, rr_map = evaluate(query["features"], query["labels"], gallery["features"], gallery["labels"],
                                  re_ranking=rr)
        self.logger.info_validation(task_name, len(query["features"]), len(gallery["features"]), rr_cmc, rr_map,
                                    label="re-ranked")
        return cmc, mAP, avg_rep, (rr_cmc, rr_map)

    def inference(self, task_name: str, query_loader, gallery_loader, device: str = "cpu", **kwargs) -> Dict:
        """``{query_id: {gallery_id: similarity}}`` as in ``methods/baseline.py:279-303`` (one GEMM, not Q of them)."""
        from ..ops.rank import similarity
        g = self._features(gallery_loader)["features"]
        q = self._features(query_loader)["features"]
        self.test_cnt += len(g) + len(q)
        sim = similarity(q, g).cpu().numpy()
        return {qi: {gi: sim[qi, gi] for gi in range(sim.shape[1])} for qi in range(sim.shape[0])}


class ServerModule(_Actor):
    def __init__(self, server_name: str, model: ModelModule, operator: OperatorModule, ckpt_root: str,
                 store: Optional[CheckpointStore] = None, comm=None, **kwargs):
        self.server_name = self.name = server_name
        self.model = model
        self.operator = operator
        self.comm = comm
        for n, p in kwargs.items():
            setattr(self, n, p)
        self.store = store if store is not None else CheckpointStore(ckpt_root, asynchronous=False)
        self.clients: Dict[str, Any] = {}
        self.logger = Logger(self.server_name)
        self.operator.logger = self.logger
        self.logger.info("Startup successfully.")

    def register_client(self, client_name: str) -> bool:
        if client_name in self.clients:
            self.logger.warn(f"'{client_name}' has already registered in server.")
            return False
        self.clients[client_name] = self.init_client_state()
        self.logger.info(f"'{client_name}' register succeed in server.")
        return True

    def unregister_client(self, client_name: str) -> bool:
        if client_name in self.clients:
            self.clients.pop(client_name)
            self.logger.info(f"'{client_name}' unregister succeed in server.")
            return True
        self.logger.warn(f"'{client_name}' is not registered in server.")
        return False

    def calculate(self) -> Any:
        return None

    def init_client_state(self) -> Any:
        return None

    def set_client_incremental_state(self, client_name: str, client_state: Dict) -> None:
        return None

    def set_client_integrated_state(self, client_name: str, client_state: Dict) -> None:
        return None

    def get_dispatch_incremental_state(self, client_name: str) -> Optional[Dict]:
        return None

    def get_dispatch_integrated_state(self, client_name: str) -> Optional[Dict]:
        return None


def _bind_loader(loader, model: ModelModule) -> None:
    """Point a :class:`DeviceBatchLoader` at the model's device / compute dtype (no-op for torch DataLoaders)."""
    if hasattr(loader, "to") and hasattr(loader, "augment"):
        # bf16 models get bf16 NHWC batches straight out of the fused augmentation kernel (the first convolution
        # would cast its input to bf16 anyway)
        loader.to(model.device, model.compute_dtype if model.device.type == "cuda" else torch.float32)
        loader.device_generator = model.rng

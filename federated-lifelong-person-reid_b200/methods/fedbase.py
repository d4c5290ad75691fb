"""Shared machinery of the federated methods: symmetric upload slots + collective aggregation.

Every federated plug-in follows the same device-resident exchange (SURVEY §7.1):

* a client *uploads* by copying the upload-prefix of its parameter arena into its slot of the symmetric ``up``
  buffer (one D2D copy; the reference clones every tensor to the CPU and ``torch.save``s it twice);
* ``server.calculate()`` is ONE fused peer-memory kernel (``FedComm.reduce_bcast``) that forms the
  ``train_cnt``-weighted mean of *every registered client's last upload* (stale uploads of offline clients included,
  exactly like ``methods/fedavg.py:386-397``) and leaves the result in the ``glob`` buffer of every rank;
* dispatch to a local client is a D2D copy from ``glob`` (incremental) or from the server replica (first contact).

The dict payloads of the reference protocol are still produced (as named views) so that the
``{round}-{src}-{dst}.ckpt`` payload checkpoints keep their schema.
"""
from __future__ import annotations

import math
from typing import Any, Dict, List, Optional

import torch

from ..ops import fused as fops
from ..ops import layer as lops
from ..runtime.modules import ClientModule, ModelModule, ServerModule


def _reprefix(state: Dict[str, torch.Tensor], prefix: str) -> Dict[str, torch.Tensor]:
    """Re-key a ``net.*`` state dict with ``prefix`` (``"net."`` or ``""``); accepts either form as input."""
    return {prefix + (k[4:] if k.startswith("net.") else k): v for k, v in state.items()}


class FedClient(ClientModule):
    """Client side of the FedAvg-family exchange."""

    default_ckpt_name = "fedavg_model"
    upload_key = "incremental_model_params"
    integrated_key = "integrated_model_params"
    # FedAvg enumerates the ``ModelModule`` wrapper (keys ``net.*``, methods/fedavg.py:232-242); FedProx / FedCurv
    # enumerate ``model.net`` (bare keys, methods/fedprox.py:321-331, fedcurv.py:395-411)
    payload_prefix = "net."

    def __init__(self, client_name, model, operator, ckpt_root, model_ckpt_name=None, **kwargs):
        super().__init__(client_name, model, operator, ckpt_root, model_ckpt_name, **kwargs)
        self.model.operator = operator
        if not self.model_ckpt_name:
            self.model_ckpt_name = self.default_ckpt_name

    # ---- symmetric buffers --------------------------------------------------------------------------------------
    @classmethod
    def declare_buffers(cls, comm, model, token_numel: int = 0) -> None:
        """Symmetric allocations – executed identically on every rank (also ranks hosting no client)."""
        n = cls._upload_numel(model)
        if model.device.type == "cuda":
            lops.enabled("apply", model.device)           # one-time isolated self-check of the dispatch kernel, up front
        comm.alloc_client_buffer("up", n)
        comm.alloc_client_buffer("cnt", 4)
        comm.alloc_rank_buffer("glob", n)

    @staticmethod
    def _upload_numel(model) -> int:
        a = model.arena
        return a.prefix_numel if a.prefix_numel else a.numel

    def upload_numel(self) -> int:
        return self._upload_numel(self.model)

    def _named_prefix(self, flat: torch.Tensor) -> Dict[str, torch.Tensor]:
        """Named views of the upload prefix of a flat buffer, keyed like the reference's payload."""
        a = self.model.arena
        out = {}
        for name, seg in a.segments.items():
            if seg.offset + seg.numel <= flat.numel():
                out[self.payload_prefix + name] = a.view(flat, name)
        return out

    def _full_state(self) -> Dict[str, torch.Tensor]:
        return _reprefix(self.model.full_state(), self.payload_prefix)

    # ---- protocol -----------------------------------------------------------------------------------------------
    def get_incremental_state(self, **kwargs) -> Dict:
        n = self.upload_numel()
        slot = self.comm.client_view("up", self.client_id)
        slot.copy_(self.model.arena.master[:n])
        self.comm.client_view("cnt", self.client_id).fill_(float(self.train_cnt))
        return {"train_cnt": self.train_cnt, self.upload_key: self._named_prefix(slot)}

    def get_integrated_state(self, **kwargs) -> Dict:
        return {"train_cnt": self.train_cnt, self.integrated_key: self._full_state()}

    def apply_global(self, flat: torch.Tensor, p_old: Optional[torch.Tensor] = None, snap_mode: int = 0) -> None:
        """Overwrite the upload-prefix of the arena with ``flat`` (the aggregated parameters). On CUDA one kernel writes
        the fp32 master, the bf16 compute copy and - FedProx - the proximal anchor ``p_old`` (``snap_mode`` 1: the
        weights being replaced, 2: the incoming ones) in the same pass (``ops.layer.apply_global``)."""
        a = self.model.arena
        n = flat.numel()
        if flat.is_cuda and lops.enabled("apply", flat.device):
            lops.apply_global(flat, a.master, a.shadow, p_old, snap_mode)
            if n < a.numel and p_old is not None and snap_mode:
                p_old[n:].copy_(a.master[n:])            # (the tail of the arena is not part of the exchange)
            return
        if p_old is not None and snap_mode == 1:
            p_old.copy_(a.master)
        a.master[:n].copy_(flat)
        if p_old is not None and snap_mode == 2:
            p_old.copy_(a.master)
        a.refresh_shadow()

    def update_by_incremental_state(self, state: Dict, **kwargs) -> Any:
        self.train_cnt = self.test_cnt = 0
        self.before_global_update()
        if "_flat" in state:
            self.apply_global(state["_flat"])
        else:
            self.model.arena.from_dict({k[4:] if k.startswith("net.") else k: v
                                        for k, v in state[self.upload_key].items()})
        self.logger.info("Update model succeed by incremental state from server.")

    def update_by_integrated_state(self, state: Dict, **kwargs) -> Any:
        self.train_cnt = self.test_cnt = 0
        self.before_global_update()
        self.model.load_full_state(_reprefix(state[self.integrated_key], "net."))
        self.logger.info("Update model succeed by integrated state from server.")

    def before_global_update(self) -> None:
        pass

    def after_epoch(self, output: Dict) -> None:
        self.train_cnt += output["data_count"]              # methods/fedavg.py:298


_SERVER_OPT_KEYS = {"sgd": {"lr": None, "momentum": 0.0}}
_SERVER_OPT_KEYS.update({name: {"lr": None, "beta1": 0.9, "beta2": 0.99, "tau": 1e-3}
                         for name in ("adagrad", "adam", "yogi")})


def parse_server_opt(cfg: Optional[Dict]) -> Optional[Dict[str, Any]]:
    """Validate the ``server: server_opt:`` block, e.g. ``{name: adam, lr: 0.01, beta1: 0.9, beta2: 0.99, tau: 0.001}``,
    and return it with the defaults filled in (``None``: no block, plain FedAvg replacement of the replica).
    ``sgd`` takes ``lr`` and ``momentum``; ``adagrad`` / ``adam`` / ``yogi`` take ``lr``, ``beta1``, ``beta2`` (unused by
    ``adagrad``) and ``tau``. Raises ``ValueError`` on an unknown name or key, a missing or non-positive ``lr``, a
    ``momentum`` / ``beta1`` / ``beta2`` outside ``[0, 1)`` or a non-positive ``tau``."""
    if cfg is None:
        return None
    if not isinstance(cfg, dict):
        raise ValueError(f"server_opt must be a mapping, got {cfg!r}")
    name = cfg.get("name")
    if name not in _SERVER_OPT_KEYS:
        raise ValueError(f"server_opt: unknown name {name!r} (one of {sorted(_SERVER_OPT_KEYS)})")
    allowed = _SERVER_OPT_KEYS[name]
    unknown = sorted(set(cfg) - set(allowed) - {"name"})
    if unknown:
        raise ValueError(f"server_opt: unknown key(s) {unknown} for {name!r} (allowed: {sorted(allowed)})")
    if "lr" not in cfg:
        raise ValueError("server_opt: lr is required")
    out: Dict[str, Any] = {"name": name}
    for key, default in allowed.items():
        try:
            out[key] = float(cfg.get(key, default))
        except (TypeError, ValueError):
            raise ValueError(f"server_opt: {key} must be a number, got {cfg.get(key)!r}") from None
    if not out["lr"] > 0:
        raise ValueError(f"server_opt: lr must be > 0, got {out['lr']}")
    for key in ("momentum", "beta1", "beta2"):
        if key in out and not 0 <= out[key] < 1:
            raise ValueError(f"server_opt: {key} must be in [0, 1), got {out[key]}")
    if "tau" in out and not out["tau"] > 0:
        raise ValueError(f"server_opt: tau must be > 0, got {out['tau']}")
    return out


def parse_aggregator(cfg: Optional[Dict]) -> Optional[Dict[str, Any]]:
    """Validate the ``server: aggregator:`` block, ``{name: median}`` or ``{name: trimmed_mean, beta: 0.2}``, and return
    it with the default ``beta`` (0.1) filled in (``None``: no block, the ``train_cnt``-weighted mean). ``beta`` must be
    a finite number with ``0 <= beta < 0.5``. Raises ``ValueError`` on an unknown name or key or a bad ``beta``."""
    if cfg is None:
        return None
    if not isinstance(cfg, dict):
        raise ValueError(f"aggregator must be a mapping, got {cfg!r}")
    name = cfg.get("name")
    allowed = {"median": set(), "trimmed_mean": {"beta"}}
    if name not in allowed:
        raise ValueError(f"aggregator: unknown name {name!r} (one of {sorted(allowed)})")
    unknown = sorted(set(cfg) - allowed[name] - {"name"})
    if unknown:
        raise ValueError(f"aggregator: unknown key(s) {unknown} for {name!r} (allowed: {sorted(allowed[name])})")
    if name == "median":
        return {"name": name}
    beta = cfg.get("beta", 0.1)
    if isinstance(beta, bool) or not isinstance(beta, (int, float)):
        raise ValueError(f"aggregator: beta must be a number, got {beta!r}")
    beta = float(beta)
    if not (math.isfinite(beta) and 0 <= beta < 0.5):
        raise ValueError(f"aggregator: beta must be finite and in [0, 0.5), got {beta}")
    return {"name": name, "beta": beta}


def trim_count(beta: float, K: int) -> int:
    """Values cut from each end by ``trimmed_mean`` over ``K`` uploads: ``floor(beta * K)``, the cut of
    ``scipy.stats.trim_mean``."""
    return int(beta * K)


class FedServer(ServerModule):
    """Server role of the FedAvg-family exchange (replicated on every rank).

    ``server_opt`` (optional, :func:`parse_server_opt`): instead of overwriting the replica with the aggregated mean,
    ``calculate()`` takes one server-optimizer step toward it (FedAvgM / FedAdagrad / FedAdam / FedYogi,
    ``ops.fused.server_opt_step``). ``glob`` is bitwise identical on every rank, so the replicated step keeps the replicas
    (and their moments ``m`` / ``v``) identical without any extra communication.

    ``aggregator`` (optional, :func:`parse_aggregator`): ``glob`` is the coordinate-wise median or trimmed mean of the
    uploads (unweighted, ``FedComm.reduce_robust``) instead of their ``train_cnt``-weighted mean. It has no state, and
    ``server_opt`` steps toward it like toward the mean."""

    upload_key = "incremental_model_params"
    integrated_key = "integrated_model_params"
    payload_prefix = "net."

    def __init__(self, server_name, model, operator, ckpt_root, server_opt: Optional[Dict] = None,
                 aggregator: Optional[Dict] = None, **kwargs):
        super().__init__(server_name, model, operator, ckpt_root, **kwargs)
        self.client_ids: Dict[str, int] = {}
        self.uploaded: List[int] = []                       # client ids with a valid upload slot (insertion order)
        self.server_opt = parse_server_opt(server_opt)
        self.aggregator = parse_aggregator(aggregator)
        self.opt_m: Optional[torch.Tensor] = None           # server-optimizer moments, fp32, allocated on first use
        self.opt_v: Optional[torch.Tensor] = None

    def bind_client(self, client_name: str, client_id: int) -> None:
        self.client_ids[client_name] = client_id

    def set_client_incremental_state(self, client_name: str, client_state: Optional[Dict]) -> None:
        """``client_state`` is ``None`` for clients hosted on another rank: their slot is read over NVLink."""
        if client_name not in self.clients:
            self.logger.warn(f"Collect incremental state failed from unregistered client {client_name}.")
            return
        self.clients[client_name] = client_state if client_state is not None else {"remote": True}
        cid = self.client_ids[client_name]
        if cid not in self.uploaded:
            self.uploaded.append(cid)
        self.logger.info(f"Collect incremental state successfully from client {client_name}.")

    set_client_integrated_state = set_client_incremental_state

    def aggregate(self) -> Optional[torch.Tensor]:
        if not self.uploaded:
            return None
        agg = self.aggregator
        if agg is not None:
            b = trim_count(agg["beta"], len(self.uploaded)) if agg["name"] == "trimmed_mean" else 0
            self.comm.reduce_robust("up", "glob", self.uploaded, agg["name"], b)
            return self.comm.rank_view("glob")
        self.comm.reduce_bcast("up", "glob", self.uploaded, cnt="cnt")
        return self.comm.rank_view("glob")

    def calculate(self) -> Any:
        glob = self.aggregate()
        if glob is None:
            return
        a = self.model.arena
        if self.server_opt is None:
            a.master[:glob.numel()].copy_(glob)
            a.refresh_shadow()
            return
        n, o = glob.numel(), self.server_opt
        if self.opt_m is None:
            self.opt_m = torch.zeros(n, dtype=torch.float32, device=a.device)
            if o["name"] != "sgd":
                self.opt_v = torch.zeros(n, dtype=torch.float32, device=a.device)
        # (the arena tail beyond the upload prefix never changes here, so its bf16 copy stays current)
        fops.server_opt_step(o["name"], a.master[:n], glob, self.opt_m, self.opt_v, lr=o["lr"],
                             momentum=o.get("momentum", 0.0), beta1=o.get("beta1", 0.9), beta2=o.get("beta2", 0.99),
                             tau=o.get("tau", 1e-3), x_bf16=None if a.shadow is None else a.shadow[:n])

    def resume_extra(self) -> Dict[str, Any]:
        """The server-optimizer moments (replicated like the replica itself); ``{}`` without ``server_opt``."""
        if self.server_opt is None:
            return {}
        return {"server_opt_m": self.opt_m, "server_opt_v": self.opt_v}

    def load_resume_extra(self, extra: Dict[str, Any]) -> None:
        if self.server_opt is None:
            return
        dev = self.model.arena.device
        m, v = extra.get("server_opt_m"), extra.get("server_opt_v")
        self.opt_m = None if m is None else m.to(dev, torch.float32).clone()
        self.opt_v = None if v is None else v.to(dev, torch.float32).clone()

    def _named_global(self) -> Dict[str, torch.Tensor]:
        a = self.model.arena
        n = self.comm.bufs["glob"].n if self.comm is not None and "glob" in self.comm.bufs else a.numel
        return {self.payload_prefix + name: a.view(a.master, name) for name, seg in a.segments.items()
                if seg.offset + seg.numel <= n}

    def get_dispatch_incremental_state(self, client_name: str) -> Dict:
        a = self.model.arena
        n = self.comm.bufs["glob"].n
        return {self.upload_key: self._named_global(), "_flat": a.master[:n]}

    def get_dispatch_integrated_state(self, client_name: str) -> Dict:
        return {self.integrated_key: _reprefix(self.model.full_state(), self.payload_prefix)}


def strip_private(state: Optional[Dict]) -> Optional[Dict]:
    """Drop engine-internal handles (keys starting with ``_``) before a payload is checkpointed."""
    if state is None:
        return None
    return {k: v for k, v in state.items() if not (isinstance(k, str) and k.startswith("_"))}

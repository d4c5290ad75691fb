"""``si`` - Synaptic Intelligence (Zenke, Poole and Ganguli, ICML 2017), local-only continual learning.

Per trainable arena element ``k``:

* every optimizer step adds ``W_k += -g_k * (p_k_after - p_k_before)``, the path integral of the loss gradient
  ``g`` (``a.grad``: without the penalty, weight-decay or L1 terms) along the update the step actually applied. It is
  one more fp32 stream of the fused optimizer kernel (``omega``), with no saved copy of the weights and no extra pass;
* when ``before_train`` sees a task other than the one it tracks, the finished task is consolidated (Eq. 5, no
  clamping): ``Omega_k += W_k / ((p_k - p_old_k)^2 + xi)``, then ``p_old = p``, ``W = 0``. The first task has nothing
  to consolidate (its start point is taken when its training begins); the last task is never consolidated;
* the surrogate loss ``c * sum Omega (p - p_old)^2`` is the quadratic penalty of :class:`PenaltyModel` with
  ``Q = Omega`` (``F``) and ``R = Omega * p_old``, so ``c`` is ``lambda_penalty``.

Weight changes that are not optimizer steps (a dispatch that overwrites the net) add nothing to ``W``.
Checkpoint ``si_model``: EWC's keys (``precision_matrices`` = ``Omega``) plus ``path_integral`` (``W``)."""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch

from . import ewc
from .penalty import PenaltyModel


class Model(PenaltyModel):
    resume_attrs = PenaltyModel.resume_attrs + ("W", "task_name")
    lambda_default = 0.1

    def __init__(self, net, operator=None, si_xi: float = 1e-3, **kwargs):
        super().__init__(net, operator, **kwargs)
        if not (math.isfinite(self.lam) and self.lam >= 0.0):
            raise ValueError(f"si: lambda_penalty must be finite and >= 0, got {self.lam}")
        self.xi = float(si_xi)
        if not (math.isfinite(self.xi) and self.xi > 0.0):
            raise ValueError(f"si: si_xi must be finite and > 0, got {self.xi}")
        self.W: Optional[torch.Tensor] = None            # path integral of the current task (flat, arena layout)
        self.task_name: Optional[str] = None             # task whose trajectory W integrates

    def materialize(self, device, compute_dtype="bf16", fine_tuning=None):
        super().materialize(device, compute_dtype, fine_tuning)
        self.W = self.arena.new_buffer()                 # one object for the model's life: CUDA graphs hold its address
        return self

    def install(self, optimizer) -> None:
        super().install(optimizer)
        optimizer.omega = self.W

    def switch_task(self, task_name: str) -> None:
        """Consolidate the tracked task when ``task_name`` differs from it; start tracking ``task_name``."""
        if task_name == self.task_name:
            return
        with torch.no_grad():
            if self.task_name is not None:
                d = self.arena.master - self.p_old
                self.F.add_(self.W / (d * d + self.xi))
            self.p_old.copy_(self.arena.master)
            self.W.zero_()
            self.rebuild_penalty()
        self.task_name = task_name

    def model_state(self) -> Dict:
        state = super().model_state()
        state["path_integral"] = self.arena.to_dict(self.W)
        return state

    def update_model(self, params_state: Dict) -> None:
        super().update_model(params_state)
        if self.arena is not None and "path_integral" in params_state:
            self.arena.from_dict(params_state["path_integral"], self.W)


class Operator(ewc.Operator):
    pass


class Client(ewc.Client):
    default_ckpt_name = "si_model"

    def before_train(self, task_name, tr_loader, val_loader) -> None:
        self.model.switch_task(task_name)
        self.model.install(self.operator.optimizer)

    def after_train(self, task_name, tr_loader, val_loader, output) -> None:
        pass                                             # importance comes from the trajectory, not a Fisher pass


class Server(ewc.Server):
    pass

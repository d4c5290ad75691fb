"""Flat, persistent parameter arenas and the fused optimizers that run over them.

Every client keeps its trainable state in ONE contiguous fp32 buffer (``master``), a same-shaped gradient buffer that
autograd accumulates into in place, an optional bf16 compute copy (``shadow``) refreshed by the optimizer kernel, and
the optimizer moments. Named ``nn.Parameter`` objects are *views* into the arena, so the reference's dict schemas are
reconstructed only at checkpoint / payload time (SURVEY §7.1). On CUDA, conv weights are laid out OHWI
(``channels_last``) so the wgmma implicit-GEMM kernels read them without any per-step transpose; a CPU arena keeps
the standard OIHW order, which makes the fp32 CPU path run the very same ATen kernels as the reference (the
whole-experiment golden tests rely on that).

The optimizers implement ``torch.optim.Adam`` / ``torch.optim.SGD`` semantics (``models/__init__.py:18-21``) with the
continual-learning penalty, FedSTIL L1 term and bf16 refresh fused into the same pass (``csrc/fused_ops.cu``).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Dict, Iterable, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from ..ops import fused as fops


@dataclass
class Segment:
    name: str
    offset: int
    numel: int
    shape: Tuple[int, ...]
    channels_last: bool


def _phys(t: torch.Tensor, channels_last: bool) -> torch.Tensor:
    """Flatten ``t`` in arena (physical) order."""
    if channels_last:
        return t.detach().permute(0, 2, 3, 1).reshape(-1)
    return t.detach().reshape(-1)


class ParamArena:
    def __init__(self, named_params: Sequence[Tuple[str, nn.Parameter]], device: torch.device | str,
                 shadow: bool = False, first: Optional[Callable[[str], bool]] = None):
        """``first(name) -> bool`` selects the parameters placed at the front (the upload prefix)."""
        self.device = torch.device(device)
        items = list(named_params)
        if first is not None:
            items = [it for it in items if first(it[0])] + [it for it in items if not first(it[0])]
        self.segments: Dict[str, Segment] = {}
        self.params: Dict[str, nn.Parameter] = {}
        off = 0
        self.prefix_numel = 0
        for name, p in items:
            cl = p.dim() == 4 and self.device.type == "cuda"
            n = p.numel()
            self.segments[name] = Segment(name, off, n, tuple(p.shape), cl)
            self.params[name] = p
            off += (n + 3) // 4 * 4
            if first is not None and first(name):
                self.prefix_numel = off
        self.numel = max(off, 4)
        self.master = torch.zeros(self.numel, dtype=torch.float32, device=self.device)
        self.grad = torch.zeros(self.numel, dtype=torch.float32, device=self.device)
        self.shadow = torch.zeros(self.numel, dtype=torch.bfloat16, device=self.device) if shadow else None
        self._by_id: Dict[int, Segment] = {}
        for name, p in items:
            seg = self.segments[name]
            self.master[seg.offset:seg.offset + seg.numel].copy_(_phys(p.data.to(self.device), seg.channels_last))
            p.data = self._view(self.master, seg)
            p.grad = self._view(self.grad, seg)
            self._by_id[id(p)] = seg
        self.refresh_shadow()

    # ------------------------------------------------------------------ views
    @staticmethod
    def _view(flat: torch.Tensor, seg: Segment) -> torch.Tensor:
        t = flat[seg.offset:seg.offset + seg.numel]
        if seg.channels_last:
            o, i, h, w = seg.shape
            return t.view(o, h, w, i).permute(0, 3, 1, 2)
        return t.view(seg.shape)

    def view(self, flat: torch.Tensor, name: str) -> torch.Tensor:
        return self._view(flat, self.segments[name])

    def shadow_of(self, p: torch.Tensor) -> Optional[torch.Tensor]:
        if self.shadow is None:
            return None
        seg = self._by_id.get(id(p))
        return None if seg is None else self._view(self.shadow, seg)

    def grad_of(self, p: torch.Tensor) -> Optional[torch.Tensor]:
        """The parameter's view of the flat gradient buffer (kernels may write weight gradients straight into it)."""
        seg = self._by_id.get(id(p))
        return None if seg is None else self._view(self.grad, seg)

    def refresh_shadow(self) -> None:
        if self.shadow is not None:
            fops.cast_bf16(self.master, self.shadow)

    def zero_grad(self) -> None:
        self.grad.zero_()
        for name, p in self.params.items():           # autograd may have replaced .grad (e.g. after set_to_none)
            if p.grad is None or p.grad.data_ptr() != self.grad.data_ptr() + self.segments[name].offset * 4:
                p.grad = self._view(self.grad, self.segments[name])

    def new_buffer(self, fill: float = 0.0) -> torch.Tensor:
        return torch.full((self.numel,), fill, dtype=torch.float32, device=self.device)

    # ------------------------------------------------------------------ dict <-> flat
    def to_dict(self, flat: Optional[torch.Tensor] = None, names: Optional[Iterable[str]] = None,
                device: Optional[str] = None) -> Dict[str, torch.Tensor]:
        """Standard-layout (contiguous) copies keyed by parameter name."""
        flat = self.master if flat is None else flat
        out = {}
        for name in (names if names is not None else self.segments):
            t = self._view(flat, self.segments[name]).detach().clone(memory_format=torch.contiguous_format)
            out[name] = t.to(device) if device is not None else t
        return out

    def from_dict(self, state: Dict[str, torch.Tensor], flat: Optional[torch.Tensor] = None) -> None:
        flat = self.master if flat is None else flat
        with torch.no_grad():
            for name, t in state.items():
                seg = self.segments.get(name)
                if seg is not None:
                    flat[seg.offset:seg.offset + seg.numel].copy_(_phys(t.to(self.device), seg.channels_last))
        if flat is self.master:
            self.refresh_shadow()


class ArenaOptimizer:
    """Adam / SGD over a :class:`ParamArena` in one kernel launch."""

    def __init__(self, kind: str, arena: ParamArena, lr: float = 1e-3, weight_decay: float = 0.0,
                 betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8, momentum: float = 0.0, **unused):
        if kind not in ("adam", "sgd"):
            raise ValueError(f"unknown optimizer {kind}")
        self.kind, self.arena = kind, arena
        self.defaults = {"lr": float(lr), "weight_decay": float(weight_decay), "betas": tuple(betas), "eps": float(eps),
                         "momentum": float(momentum)}
        self.lr = float(lr)
        self.m: Optional[torch.Tensor] = None
        self.v: Optional[torch.Tensor] = None
        self.step_count = 0
        # fused extras (set by the method plug-ins)
        self.Q: Optional[torch.Tensor] = None
        self.R: Optional[torch.Tensor] = None
        self.lam2 = 0.0
        self.penalty_ones = False
        self.G: Optional[torch.Tensor] = None
        self.lam1 = 0.0
        self.atten = 0.0
        self.stats: Optional[torch.Tensor] = None
        # FedSTIL ``train_l1_anchor`` (off by default): the L1 anchor is a trained tensor with its own moments
        self.anchor: Optional[torch.Tensor] = None
        self.anchor_m: Optional[torch.Tensor] = None
        self.anchor_v: Optional[torch.Tensor] = None
        # Synaptic Intelligence path integral (methods/si.py), accumulated by the step; must stay the same tensor while
        # a CUDA graph of the step is live
        self.omega: Optional[torch.Tensor] = None
        # device-resident [lr, step] (CUDA only): a captured CUDA graph of the train step stays valid across steps
        self.hyper: Optional[torch.Tensor] = None
        if arena.device.type == "cuda":
            self.hyper = torch.tensor([self.lr, 0.0], dtype=torch.float32, device=arena.device)

    @property
    def param_groups(self) -> List[dict]:           # minimal torch.optim-like surface (lr scheduling / logging)
        return [{"lr": self.lr, **{k: v for k, v in self.defaults.items() if k != "lr"}}]

    def zero_grad(self, set_to_none: bool = False) -> None:
        self.arena.zero_grad()

    def reset_state(self) -> None:
        """The reference wipes ``optimizer.state`` and restores lr after every ``train()`` (baseline.py:263-266)."""
        if self.m is not None:
            self.m.zero_()
        if self.v is not None:
            self.v.zero_()
        for buf in (self.anchor_m, self.anchor_v):
            if buf is not None:
                buf.zero_()
        self.step_count = 0
        self.lr = self.defaults["lr"]
        self.sync_hyper()

    def restore_default_lr(self) -> None:
        """Back to the configured lr (no device traffic unless a scheduler changed it)."""
        if self.lr != self.defaults["lr"]:
            self.lr = self.defaults["lr"]
            self.sync_hyper()

    def sync_hyper(self) -> None:
        """Push the host-side lr / step counter to the device copy (call after changing ``lr``)."""
        if self.hyper is not None:
            self.hyper.copy_(torch.tensor([self.lr, float(self.step_count)]), non_blocking=True)

    def step(self) -> None:
        a = self.arena
        if self.omega is not None and (self.G is not None or self.anchor is not None):
            raise ValueError("the SI path integral (omega) cannot be combined with FedSTIL's G / trained L1 anchor")
        if self.m is None and (self.kind == "adam" or self.defaults["momentum"] != 0.0):
            self.m = a.new_buffer()
        if self.v is None and self.kind == "adam":
            self.v = a.new_buffer()
        self.step_count += 1
        d = self.defaults
        if self.hyper is not None:
            self.hyper[1:2].add_(1.0)                 # captured together with the step when graphing

        n_g = self.G.numel() if self.G is not None else 0
        trained_anchor = self.anchor is not None and n_g > 0 and self.lam1 != 0.0
        fused_anchor = trained_anchor and getattr(self, "fuse_anchor", True) and (
            a.device.type == "cuda" or bool(fops._emu_libs))      # (tests: the kernel under the CPU SIMT emulator)
        if fused_anchor and self.anchor_m is None and (self.kind == "adam" or d["momentum"] != 0.0):
            self.anchor_m = torch.zeros_like(self.anchor)
        if fused_anchor and self.anchor_v is None and self.kind == "adam":
            self.anchor_v = torch.zeros_like(self.anchor)

        def launch(lo: int, hi: int, with_g: bool) -> None:
            sl = slice(lo, hi)
            anc = with_g and fused_anchor
            fops.fused_optimizer_step(
                self.kind, a.master[sl], a.grad[sl], None if self.m is None else self.m[sl],
                None if self.v is None else self.v[sl], lr=self.lr, step=self.step_count, beta1=d["betas"][0],
                beta2=d["betas"][1], eps=d["eps"], weight_decay=d["weight_decay"], momentum=d["momentum"],
                Q=None if self.Q is None else self.Q[sl], R=None if self.R is None else self.R[sl], lam2=self.lam2,
                penalty_ones=self.penalty_ones, G=self.G[sl] if with_g else None, lam1=self.lam1, atten=self.atten,
                p_bf16=None if a.shadow is None else a.shadow[sl], stats=self.stats, hyper=self.hyper,
                anchor=self.anchor[sl] if anc else None,
                anchor_m=self.anchor_m[sl] if anc and self.anchor_m is not None else None,
                anchor_v=self.anchor_v[sl] if anc and self.anchor_v is not None else None,
                omega=None if self.omega is None else self.omega[sl])

        lam1, l1_before = self.lam1, None
        if trained_anchor and not fused_anchor:
            l1_before = self._anchor_step(n_g)
            self.lam1 = 0.0                # the L1 sub-gradient is already in ``grad``; G still anchors the weight decay
        if 0 < n_g < a.numel:          # FedSTIL: only the adaptive-weight prefix carries the L1 / attention terms
            launch(0, n_g, True)
            launch(n_g, a.numel, False)
        else:
            launch(0, a.numel, n_g > 0)
        if trained_anchor and not fused_anchor:
            self.lam1 = lam1
            if l1_before is not None:
                self.stats[1:2].copy_(l1_before)

    def _anchor_step(self, n: int) -> Optional[torch.Tensor]:
        """Reference quirk (``engine_opts.train_l1_anchor``, on under ``reference_compat``): FedSTIL's
        ``initial_adaptive_weight`` is a bare ``Parameter`` whose ``requires_grad`` is never cleared, so the reference's
        optimizer trains the L1 *anchor* ``aw0`` as well (SURVEY §2.3) - its gradient is
        ``-lam1 * sign(aw - aw0) + wd * aw0``. This is the fp32 tensor-op form used on the CPU (what the golden tests run);
        on CUDA the same update is part of ``fused_opt_kernel``. ``anchor`` holds ``theta0 = atten * G + aw0``.
        Returns what ``stats[1]`` must read after the step: previous value + ``sum |aw - aw0|`` (for loss reporting)."""
        a, d = self.arena, self.defaults
        with torch.no_grad():
            p, g, anc = a.master[:n], a.grad[:n], self.anchor
            diff = p - anc
            l1 = None
            if self.stats is not None:
                l1 = self.stats[1:2] + diff.abs().sum()
            if self.hyper is not None:
                lr, step = self.hyper[0], self.hyper[1]
            else:
                lr, step = self.lr, float(self.step_count)
            # Where the loss gradient is exactly zero (inputs behind a dead ReLU) weight and anchor receive the same
            # update and stay *identical* in the reference, sign(0) = 0. Two differently fused update formulas cannot
            # promise bit-identical results, so differences at rounding level (1e-6 of a step) count as zero.
            s = torch.sign(diff) * (diff.abs() > 1e-6 * lr)
            g.add_(s, alpha=self.lam1)                                        # d/d aw
            g0 = s * (-self.lam1)                                             # d/d aw0 = -lam1 * s + wd * aw0
            g0.add_(anc - self.atten * self.G[:n], alpha=d["weight_decay"])
            if self.kind == "adam":
                if self.anchor_m is None:
                    self.anchor_m, self.anchor_v = torch.zeros_like(anc), torch.zeros_like(anc)
                b1, b2 = d["betas"]
                self.anchor_m.mul_(b1).add_(g0, alpha=1 - b1)
                self.anchor_v.mul_(b2).addcmul_(g0, g0, value=1 - b2)
                bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
                denom = self.anchor_v.sqrt() / (bc2 ** 0.5) + d["eps"]
                if isinstance(lr, torch.Tensor):
                    anc.sub_(self.anchor_m / denom * (lr / bc1))
                else:
                    anc.addcdiv_(self.anchor_m, denom, value=-lr / bc1)       # the op sequence of the fp32 CPU step
            else:
                if d["momentum"] != 0.0:
                    if self.anchor_m is None:
                        self.anchor_m = torch.zeros_like(anc)
                    self.anchor_m.mul_(d["momentum"]).add_(g0)
                    g0 = self.anchor_m
                anc.sub_(g0 * lr) if isinstance(lr, torch.Tensor) else anc.add_(g0, alpha=-lr)
        return l1


class StepLR:
    """``torch.optim.lr_scheduler.StepLR`` in its chainable form (``models/__init__.py:23-25``): every
    ``step_size``-th call multiplies the *current* lr by ``gamma``; the epoch counter survives lr resets."""

    def __init__(self, optimizer: ArenaOptimizer, step_size: int, gamma: float = 0.1, **unused):
        self.optimizer, self.step_size, self.gamma = optimizer, int(step_size), float(gamma)
        self.last_epoch = 0

    def step(self) -> None:
        self.last_epoch += 1
        if self.last_epoch % self.step_size == 0:
            self.optimizer.lr *= self.gamma
            self.optimizer.sync_hyper()

    def state_dict(self) -> dict:
        return {"last_epoch": self.last_epoch}

    def load_state_dict(self, sd: dict) -> None:
        self.last_epoch = int(sd["last_epoch"])


optimizers = {"adam": lambda arena, **kw: ArenaOptimizer("adam", arena, **kw),
              "sgd": lambda arena, **kw: ArenaOptimizer("sgd", arena, **kw)}
schedulers = {"step_lr": StepLR}

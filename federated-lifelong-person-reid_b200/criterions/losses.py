"""Loss functions with the reference's call convention ``loss(score=, feature=, target=)``.

* :class:`CrossEntropyLabelSmooth` – ``criterions/cross_entropy.py`` (the only loss any shipped config uses); on
  CUDA it is one fused kernel (log-softmax + smoothing + gradient + top-1 count) instead of a CPU one-hot scatter.
* :class:`TripletLoss` – ``criterions/triplet_loss.py`` (euclid / cosine distance matrix, hard or softmax-weighted
  mining, margin-ranking or soft-margin); the distance matrix runs on the wgmma GEMM for CUDA inputs.
* :class:`DistillKL` – ``criterions/kd_loss.py`` (dead code in the reference: never registered). Registered here
  as ``kd_loss`` because BASELINE.json names a CE+triplet+KD configuration.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops import fused as fops
from ..ops import gemm as gops


class CriterionModule(nn.Module):
    def forward(self, score, target, **kwargs):
        raise NotImplementedError


class CrossEntropyLabelSmooth(CriterionModule):
    def __init__(self, num_classes: int, epsilon: float = 0.1, **kwargs):
        super().__init__()
        for k, v in kwargs.items():
            setattr(self, k, v)
        self.num_classes = num_classes
        self.epsilon = epsilon
        self.stats: Optional[torch.Tensor] = None      # optional device accumulator [loss, top-1 hits]

    def forward(self, score, target, **kwargs):
        if score.shape[1] != self.num_classes:          # keep the reference's eps/K with K = configured classes
            logp = F.log_softmax(score.float(), dim=1)
            t = torch.zeros_like(logp).scatter_(1, target.view(-1, 1), 1.0)
            t = (1 - self.epsilon) * t + self.epsilon / self.num_classes
            return (-t * logp).mean(0).sum()
        return fops.ce_label_smooth(score, target, self.epsilon, self.stats)


def euclidean_dist(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """``tools/distance.py:9-16`` (squared euclidean, no sqrt – as in the reference)."""
    xx = x.float().pow(2).sum(1, keepdim=True)
    yy = y.float().pow(2).sum(1, keepdim=True).t()
    if x.is_cuda and x.shape[1] % 8 == 0 and not (x.requires_grad or y.requires_grad):
        xy = gops.gemm(x.to(torch.bfloat16), y.to(torch.bfloat16), out_dtype=torch.float32)
    else:
        xy = x.float() @ y.float().t()
    return xx + yy - 2 * xy


def cosine_dist(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """``tools/distance.py:19-30``."""
    x = F.normalize(x.float(), p=2, dim=1)
    y = F.normalize(y.float(), p=2, dim=1)
    return 1 - x @ y.t()


def kl_distance(feature: torch.Tensor, others: torch.Tensor) -> torch.Tensor:
    """``tools/distance.py:33-36``: ``KL(softmax(others) || softmax(feature))`` summed over all elements."""
    return F.kl_div(F.log_softmax(feature.float(), dim=-1), F.softmax(others.float(), dim=-1), reduction="sum")


class TripletLoss(CriterionModule):
    def __init__(self, margin=None, norm_feat: bool = False, hard_mining: bool = False, **kwargs):
        super().__init__()
        for k, v in kwargs.items():
            setattr(self, k, v)
        self.margin = margin
        self.norm_feat = norm_feat
        self.hard_mining = hard_mining

    @staticmethod
    def _softmax_weights(dist: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
        mx = (dist * mask).max(dim=1, keepdim=True)[0]
        e = torch.exp(dist - mx) * mask
        return e / (e.sum(dim=1, keepdim=True) + 1e-6)

    def mine(self, feature: torch.Tensor, target: torch.Tensor):
        """``(dist_ap, dist_an)``: on CUDA the Gram matrix runs on the wgmma GEMM (forward and both gradients) with
        the distance / mask / mining arithmetic fused in one kernel per direction (``csrc/loss_ops.cu``)."""
        if fops.mined_distances_supported(feature) and getattr(self, "fused", True):
            x = F.normalize(feature.float(), p=2, dim=1) if self.norm_feat else feature
            return fops.mined_distances(x, target, bool(self.norm_feat), bool(self.hard_mining))
        dist = cosine_dist(feature, feature) if self.norm_feat else euclidean_dist(feature, feature)
        n = dist.size(0)
        same = target.view(n, 1).eq(target.view(1, n))
        is_pos, is_neg = same.float(), (~same).float()
        if self.hard_mining:
            return (dist * is_pos).max(dim=1)[0], (dist * is_neg + is_pos * 1e9).min(dim=1)[0]
        ap, an = dist * is_pos, dist * is_neg
        return (ap * self._softmax_weights(ap, is_pos)).sum(1), (an * self._softmax_weights(-an, is_neg)).sum(1)

    def forward(self, feature=None, target=None, score=None, **kwargs):
        dist_ap, dist_an = self.mine(feature, target)
        y = torch.ones_like(dist_an)
        if self.margin is not None and self.margin > 0:
            return F.margin_ranking_loss(dist_an, dist_ap, y, margin=self.margin)
        loss = F.soft_margin_loss(dist_an - dist_ap, y)
        if torch.isinf(loss):
            loss = F.margin_ranking_loss(dist_an, dist_ap, y, margin=0.3)
        return loss

    __call__ = nn.Module.__call__


class DistillKL(CriterionModule):
    def __init__(self, temperature: float = 1.0, **kwargs):
        super().__init__()
        for k, v in kwargs.items():
            setattr(self, k, v)
        self.temperature = temperature

    def forward(self, y_student=None, y_teacher=None, score=None, teacher_score=None, **kwargs):
        s = y_student if y_student is not None else score
        t = y_teacher if y_teacher is not None else teacher_score
        if t is None:
            return s.new_zeros(())
        return fops.kd_kl(s, t, self.temperature)          # fused forward + gradient on CUDA (csrc/loss_ops.cu)

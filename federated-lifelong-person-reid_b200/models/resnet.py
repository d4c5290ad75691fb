"""ReID ResNets (18/34/50/101/152) with ``last_stride``, GAP and optional BNNeck.

Capability parity with ``models/resnet.py:45-344`` of the reference: the ``state_dict`` keys follow the torchvision
naming (``base.conv1``, ``base.layer{1..4}.{i}.conv{j}|bn{j}|downsample.{0,1}``, ``bottleneck``, ``classifier``) so
reference checkpoints load; train mode returns ``(cls_score, global_feat)``, eval mode returns ``global_feat``.

H100-first differences:
* the network is explicitly split into a *frozen trunk* and a *trainable head* at the first fine-tuned stage
  (the reference discovers the same cut with two ``torch.fx`` traces, ``methods/fedstil.py:258-288``);
* activations are NHWC bf16 on CUDA; the head runs on the wgmma GEMM / implicit-GEMM kernels
  (:mod:`flpr_b200.ops.gemm`) with fused batch-norm kernels, the trunk runs inference-only with folded BN;
* no network access: ImageNet weights are loaded from ``pretrained_path`` when given, else random init.
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops import fused as fops
from ..ops import gemm as gops

_SPECS: Dict[str, Tuple[str, List[int]]] = {
    "resnet18": ("basic", [2, 2, 2, 2]),
    "resnet34": ("basic", [3, 4, 6, 3]),
    "resnet50": ("bottleneck", [3, 4, 6, 3]),
    "resnet101": ("bottleneck", [3, 4, 23, 3]),
    "resnet152": ("bottleneck", [3, 8, 36, 3]),
}


def _conv(cin: int, cout: int, k: int, stride: int = 1) -> nn.Conv2d:
    return nn.Conv2d(cin, cout, kernel_size=k, stride=stride, padding=k // 2, bias=False)


class ResidualUnit(nn.Module):
    """Basic (two 3x3) or bottleneck (1x1-3x3-1x1) residual unit; attribute names match torchvision."""

    def __init__(self, kind: str, cin: int, width: int, stride: int):
        super().__init__()
        self.kind = kind
        self.stride = stride
        if kind == "basic":
            self.expansion = 1
            self.conv1, self.bn1 = _conv(cin, width, 3, stride), nn.BatchNorm2d(width)
            self.conv2, self.bn2 = _conv(width, width, 3), nn.BatchNorm2d(width)
        else:
            self.expansion = 4
            self.conv1, self.bn1 = _conv(cin, width, 1), nn.BatchNorm2d(width)
            self.conv2, self.bn2 = _conv(width, width, 3, stride), nn.BatchNorm2d(width)
            self.conv3, self.bn3 = _conv(width, width * 4, 1), nn.BatchNorm2d(width * 4)
        cout = width * self.expansion
        self.relu = nn.ReLU(inplace=True)
        self.downsample = None
        if stride != 1 or cin != cout:
            self.downsample = nn.Sequential(_conv(cin, cout, 1, stride), nn.BatchNorm2d(cout))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        identity = x if self.downsample is None else self.downsample(x)
        out = self.relu(self.bn1(self.conv1(x)))
        if self.kind == "basic":
            out = self.bn2(self.conv2(out))
        else:
            out = self.relu(self.bn2(self.conv2(out)))
            out = self.bn3(self.conv3(out))
        return self.relu(out + identity)


class ResNetTrunk(nn.Module):
    def __init__(self, kind: str, depths: Sequence[int], last_stride: int = 2):
        super().__init__()
        self.kind = kind
        self.conv1 = nn.Conv2d(3, 64, kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        cin = 64
        exp = 1 if kind == "basic" else 4
        for i, (width, depth, stride) in enumerate(zip((64, 128, 256, 512), depths, (1, 2, 2, last_stride)), 1):
            units = []
            for j in range(depth):
                units.append(ResidualUnit(kind, cin, width, stride if j == 0 else 1))
                cin = width * exp
            setattr(self, f"layer{i}", nn.Sequential(*units))
        self.out_channels = cin
        self.gap = nn.AdaptiveAvgPool2d(1)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)

    STAGES = ("stem", "layer1", "layer2", "layer3", "layer4")

    def run_stages(self, x: torch.Tensor, start: int = 0, stop: int = 5) -> torch.Tensor:
        for i in range(start, stop):
            if i == 0:
                x = self.maxpool(self.relu(self.bn1(self.conv1(x))))
            else:
                x = getattr(self, f"layer{i}")(x)
        return x

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        x = self.run_stages(x)
        return self.gap(x).flatten(1)


def _init_kaiming(m: nn.Module) -> None:       # strong-baseline style init used by the reference's BNNeck head
    if isinstance(m, nn.Linear):
        nn.init.kaiming_normal_(m.weight, a=0, mode="fan_out")
        if m.bias is not None:
            nn.init.zeros_(m.bias)
    elif isinstance(m, (nn.BatchNorm1d, nn.BatchNorm2d)) and m.affine:
        nn.init.ones_(m.weight)
        nn.init.zeros_(m.bias)


class ResNetReID(nn.Module):
    thread_safe_rng = True        # no dropout / stochastic depth: forward never draws from the default generator

    def __init__(self, model_name: str, num_classes: int = 1000, last_stride: int = 2, neck: str = "no",
                 pretrained_path: Optional[str] = None, **kwargs):
        super().__init__()
        for k, v in kwargs.items():                      # unknown config keys become attributes (resnet.py:259-260)
            setattr(self, k, v)
        if model_name not in _SPECS:
            raise ValueError(f"No model named {model_name} for generating.")
        kind, depths = _SPECS[model_name]
        self.model_name, self.num_classes, self.neck = model_name, num_classes, neck
        self.base = ResNetTrunk(kind, depths, last_stride)
        self.in_planes = self.base.out_channels
        self.gap = nn.AdaptiveAvgPool2d(1)
        if neck == "no":
            self.classifier = nn.Linear(self.in_planes, num_classes)
        elif neck == "bnneck":
            self.bottleneck = nn.BatchNorm1d(self.in_planes)
            self.bottleneck.bias.requires_grad_(False)
            self.classifier = nn.Linear(self.in_planes, num_classes, bias=False)
            _init_kaiming(self.bottleneck)
            nn.init.normal_(self.classifier.weight, std=0.001)
        else:
            raise ValueError(f"Mismatched neck type for {neck}.")
        if pretrained_path and os.path.exists(pretrained_path):
            sd = torch.load(pretrained_path, map_location="cpu")
            sd = {k: v for k, v in sd.items() if not k.startswith("fc.")}
            self.base.load_state_dict(sd, strict=False)
        self.head_start = 5          # index into ResNetTrunk.STAGES where the trainable head begins (5 = neck only)

    # ---------------------------------------------------------------- trunk / head split
    def configure_split(self, fine_tuning: Optional[Sequence[str]]) -> int:
        """The head starts at the first trunk stage that contains a fine-tuned sub-module."""
        start = 5
        if not fine_tuning:
            start = 0
        else:
            for name in fine_tuning:
                if name == "base" or name.startswith("base.conv1") or name.startswith("base.bn1"):
                    start = 0
                for i in range(1, 5):
                    if name == f"base.layer{i}" or name.startswith(f"base.layer{i}."):
                        start = min(start, i)
        self.head_start = start
        return start

    def forward_trunk(self, x: torch.Tensor) -> torch.Tensor:
        """Frozen part: input image batch -> feature map at the cut ("prototype" in FedSTIL terms).
        On CUDA with a bf16 fast head the frozen stages run on the wgmma kernels too (:class:`NativeTrunk`) - in
        train mode with batch-statistic BN and running-stat updates, which is what the reference's ``model.train()``
        does to the whole net for every method but FedSTIL (``methods/baseline.py:38``, ``models/resnet.py:229-241``)."""
        nt = getattr(self, "_native_trunk", None)
        if nt is not None and x.is_cuda and nt.supported(tuple(x.shape)):
            return nt(x)
        return self.base.run_stages(x, 0, self.head_start)

    def forward_head(self, fmap: torch.Tensor):
        """Trainable part: feature map at the cut -> ``(cls_score, global_feat)`` / ``global_feat``."""
        if fmap.is_cuda and getattr(self, "_fast_head", None) is not None:
            return self._fast_head(fmap)
        x = self.base.run_stages(fmap, self.head_start, 5)
        global_feat = x.mean(dim=(2, 3)) if x.dim() == 4 else x
        return self._neck(global_feat)

    def _neck(self, global_feat: torch.Tensor):
        feat = self.bottleneck(global_feat) if self.neck == "bnneck" else global_feat
        if self.training:
            return self.classifier(feat), global_feat
        return global_feat

    def forward(self, x: torch.Tensor):
        return self.forward_head(self.forward_trunk(x))

    def prototype_shape(self, img_size: Sequence[int]) -> Tuple[int, int, int]:
        """(C, H, W) of the feature map at the cut for an ``img_size`` input."""
        h, w = int(img_size[0]), int(img_size[1])
        if self.head_start == 0:
            return 3, h, w
        h, w = (h + 1) // 2, (w + 1) // 2
        h, w = (h + 1) // 2, (w + 1) // 2
        c = 64
        exp = 1 if self.base.kind == "basic" else 4
        for i in range(1, self.head_start):
            c = (64, 128, 256, 512)[i - 1] * exp
            if i >= 2:
                h, w = (h + 1) // 2, (w + 1) // 2
        return c, h, w


# ------------------------------------------------------------------------------------------------- fast head
class FastResNetHead:
    """wgmma execution of ``layer{k..4}`` + GAP + BNNeck + classifier over NHWC bf16 activations.

    Shares the ``nn.Parameter`` objects of the wrapped model (weights must be in ``channels_last`` memory format so
    that the OHWI view is contiguous) and an optional bf16 shadow provider ``shadow(param) -> bf16 tensor`` kept in
    sync by the fused optimizer. Stride-2 convolutions that need gradients run on the same kernels
    (``ops.gemm.conv_stride2``); only shapes outside the implicit-GEMM tiling constraints (feature maps whose width is
    not a power of two <= 128, channels not a multiple of 64) use the cuDNN fallback.
    """

    def __init__(self, model: ResNetReID, shadow=None, grad_slot=None):
        self.m = model
        self.shadow = shadow or (lambda p: None)
        self.grad_slot = grad_slot or (lambda p: None)      # param -> its view of the (zeroed) arena gradient

    # conv weight as [Cout, KH, KW, Cin] without copying (channels_last storage)
    @staticmethod
    def _ohwi(w: torch.Tensor) -> torch.Tensor:
        v = w.permute(0, 2, 3, 1)
        return v if v.is_contiguous() else v.contiguous()

    @staticmethod
    def _weight_of(layer: nn.Module):
        """``(weight, kernel, stride)`` of a convolution / linear leaf. Plain ``nn.Conv2d`` / ``nn.Linear`` (also
        parametrized ones: fedstil-atten's ``weight`` is ``gw_stack @ atten + aw``) expose ``.weight``; FedWeIT's
        decomposed layers compose ``theta = mask (.) sw + aw + sum_k atten_k aw_kb[..., k]`` on access
        (``methods/fedweit.py``). A composed weight is an autograd tensor: the native conv / GEMM returns its fp32
        gradient to autograd, which carries it on into ``aw`` / ``mask`` / ``atten``."""
        if hasattr(layer, "theta"):
            w = layer.theta(layer.training)
            k = w.shape[-1] if w.dim() == 4 else 1
            s = int(layer.stride[0]) if getattr(layer, "is_conv", False) else 1
            return w, k, s
        w = layer.weight
        if w.dim() == 4:
            return w, layer.kernel_size[0], layer.stride[0]
        return w, 1, 1

    def _shadow_of(self, w: torch.Tensor):
        """bf16 compute copy of ``w``: the optimizer-maintained arena shadow of a parameter, or the bf16 twin that a
        fused weight composition wrote next to its fp32 result (``ops.layer.compose_weight``)."""
        sh = self.shadow(w)
        return sh if sh is not None else getattr(w, "_flpr_bf16", None)

    def _conv(self, x: torch.Tensor, conv: nn.Module, want_stats: bool = False):
        """x: [N,H,W,C] bf16 -> [N,H',W',Cout] bf16 (``(y, col_part)`` with ``want_stats``: fused BN statistics)"""
        w, k, s = self._weight_of(conv)
        sh = self._shadow_of(w)
        if sh is None and not w.requires_grad and x.is_cuda and isinstance(w, nn.Parameter):
            sh = self._frozen_bf16(w)
        if getattr(conv, "bias", None) is not None:
            raise NotImplementedError("convolutions with a bias are not covered by the fast head")
        n, h, wd, c = x.shape
        gs = self.grad_slot(w)
        if k == 1 and s == 1:
            w2 = self._ohwi(w).reshape(w.shape[0], c)
            s2 = self._ohwi(sh).reshape(w.shape[0], c) if sh is not None else None
            g2 = self._ohwi(gs).reshape(w.shape[0], c) if gs is not None else None
            if want_stats:
                y, part = gops.linear(x.reshape(-1, c), w2, s2, g2, True)
                return y.view(n, h, wd, -1), part
            return gops.linear(x.reshape(-1, c), w2, s2, g2).view(n, h, wd, -1)
        if k == 3 and s == 1 and c % 64 == 0 and 128 % wd == 0 and ((h * wd <= 128 and 128 % (h * wd) == 0)
                                                                   or (h * wd > 128 and h % (128 // wd) == 0)):
            return gops.conv3x3(x, self._ohwi(w), self._ohwi(sh) if sh is not None else None,
                                self._ohwi(gs) if gs is not None else None, want_stats)
        if not (torch.is_grad_enabled() and (w.requires_grad or x.requires_grad)) and \
                gops.conv_supported(h, wd, c, k, s):
            # forward-only (frozen stage, or no_grad): any stride / kernel size the implicit GEMM covers
            wb = self._ohwi(sh if sh is not None else self._frozen_bf16(w))
            ho, wo = (h + 2 * (k // 2) - k) // s + 1, (wd + 2 * (k // 2) - k) // s + 1
            part = gops.col_part_buffer(n * ho * wo, w.shape[0], x.device) if want_stats else None
            y = gops.conv_nhwc(x, wb, padding=k // 2, stride=s, col_part=part)
            return (y, part) if want_stats else y
        if s == 2 and k in (1, 3) and gops.conv_s2_supported(h, wd, c, w.shape[0], k):
            # strided conv that needs a gradient (``last_stride: 2``, or a head cut above layer4): forward with TMA
            # element strides, dgrad / wgrad through the stride-1 kernels on the zero-stuffed output gradient
            wv = self._ohwi(w)
            return gops.conv_stride2(x, wv, self._ohwi(sh) if sh is not None else None,
                                     self._ohwi(gs) if gs is not None else None, want_stats)
        # library fallback (shapes outside the implicit-GEMM tiling constraints)
        y = F.conv2d(x.permute(0, 3, 1, 2), (sh if sh is not None else w.to(torch.bfloat16)) if not w.requires_grad
                     else w.to(torch.bfloat16), stride=s, padding=k // 2)
        y = y.permute(0, 2, 3, 1).contiguous()
        return (y, None) if want_stats else y

    # bf16 channels_last copies of FROZEN weights (not in the arena, so no optimizer-maintained shadow exists);
    # refreshed when the parameter is overwritten in place (first-contact dispatch, checkpoint restore)
    def _frozen_bf16(self, w: torch.Tensor) -> torch.Tensor:
        if not isinstance(w, nn.Parameter):             # a composed (temporary) weight: nothing to cache
            wb = w.detach().to(torch.bfloat16)
            return wb.contiguous(memory_format=torch.channels_last) if wb.dim() == 4 else wb
        cache = self.__dict__.setdefault("_frozen_cache", {})
        key = id(w)
        hit = cache.get(key)
        if hit is not None and hit[0] == w._version and hit[1] == w.data_ptr():
            return hit[2]
        with torch.no_grad():
            wb = w.detach().to(torch.bfloat16)
            if wb.dim() == 4:
                wb = wb.contiguous(memory_format=torch.channels_last)
        cache[key] = (w._version, w.data_ptr(), wb)
        return wb

    def _conv_bn(self, x: torch.Tensor, conv: nn.Conv2d, bn: nn.BatchNorm2d, relu: bool,
                 residual: Optional[torch.Tensor] = None) -> torch.Tensor:
        """conv -> batch-norm (-> +residual) (-> ReLU). In training mode the batch statistics come out of the
        convolution's epilogue (fp32 accumulators), so the separate statistics pass over the activation disappears."""
        if bn.training and x.is_cuda and self.fuse_bn_stats:
            y, part = self._conv(x, conv, True)
            return self._bn(y, bn, relu, residual, part)
        return self._bn(self._conv(x, conv), bn, relu, residual)

    fuse_bn_stats = True

    def _bn(self, x: torch.Tensor, bn: nn.BatchNorm2d, relu: bool, residual: Optional[torch.Tensor] = None,
            pre_part: Optional[torch.Tensor] = None):
        n, h, w, c = x.shape
        res2 = residual.reshape(-1, c) if residual is not None else None
        y = fops.batch_norm_nhwc(x.reshape(-1, c), bn.weight, bn.bias, bn.running_mean, bn.running_var,
                                 training=bn.training, eps=bn.eps, momentum=bn.momentum or 0.1, relu=relu,
                                 residual=res2, pre_part=pre_part,
                                 grad_slots=(self.grad_slot(bn.weight), self.grad_slot(bn.bias)))
        self._count(bn)
        return y.view(n, h, w, c)

    # ``num_batches_tracked`` bookkeeping: one tiny kernel per BN layer per step. A training loop that knows its step
    # count sets ``count_batches = False`` and calls :meth:`add_batches` once per epoch instead.
    count_batches = True

    def _count(self, bn) -> None:
        if self.count_batches and bn.training and bn.num_batches_tracked is not None:
            bn.num_batches_tracked += 1

    def batch_norms(self):
        m = self.m
        out = [b for i in range(max(m.head_start, 1), 5) for b in getattr(m.base, f"layer{i}").modules()
               if isinstance(b, (nn.BatchNorm1d, nn.BatchNorm2d))]
        if m.neck == "bnneck":
            out.append(m.bottleneck)
        return out

    def add_batches(self, n: int) -> None:
        for bn in self.batch_norms():
            if bn.num_batches_tracked is not None:
                bn.num_batches_tracked += int(n)

    def _unit(self, x: torch.Tensor, u: ResidualUnit) -> torch.Tensor:
        identity = x
        if u.downsample is not None:
            identity = self._conv_bn(x, u.downsample[0], u.downsample[1], relu=False)
        out = self._conv_bn(x, u.conv1, u.bn1, relu=True)
        if u.kind == "basic":
            return self._conv_bn(out, u.conv2, u.bn2, relu=True, residual=identity)
        out = self._conv_bn(out, u.conv2, u.bn2, relu=True)
        return self._conv_bn(out, u.conv3, u.bn3, relu=True, residual=identity)

    def __call__(self, fmap: torch.Tensor):
        m = self.m
        # fmap is logical NCHW (any memory format); channels_last storage makes this permute a free view
        x = fmap.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)
        for i in range(max(m.head_start, 1), 5):
            for u in getattr(m.base, f"layer{i}"):
                x = self._unit(x, u)
        n, h, w, c = x.shape
        global_feat = fops.global_avg_pool_nhwc(x.view(n, h * w, c))                 # fp32 [N, C]
        if m.neck == "bnneck":
            bn = m.bottleneck
            feat = fops.batch_norm_nhwc(global_feat.to(torch.bfloat16), bn.weight, bn.bias, bn.running_mean,
                                        bn.running_var, training=bn.training, eps=bn.eps, momentum=bn.momentum or 0.1,
                                        grad_slots=(self.grad_slot(bn.weight), self.grad_slot(bn.bias)))
            self._count(bn)
        else:
            feat = global_feat.to(torch.bfloat16)
        if not m.training:
            return global_feat
        w = self._weight_of(m.classifier)[0]
        score = gops.linear(feat, w, self._shadow_of(w), self.grad_slot(w))
        if m.classifier.bias is not None:
            score = score + m.classifier.bias.to(score.dtype)
        return score, global_feat


class NativeTrunk(FastResNetHead):
    """The frozen stages (stem + ``layer1..k-1``) on the wgmma kernels, forward only - nothing in them is trainable
    and their input does not require grad, so no autograd graph is built. ``model.train()``: every BatchNorm
    normalises with the batch statistics that the producing convolution's epilogue emitted and updates its running
    statistics (``bn_finalize``); ``model.eval()``: running statistics (``affine_act``).

    Stem: the 7x7 / 2 convolution runs as a 4x4 convolution over 2x2 space-to-depth cells (``ops.gemm.stem_conv``),
    then BN + ReLU, then the NHWC max-pool kernel. Strided 3x3 / 1x1 convolutions use TMA element strides."""

    def __init__(self, model: ResNetReID):
        super().__init__(model, None, None)
        self._stem_cache = None

    def supported(self, shape) -> bool:
        cache = self.__dict__.setdefault("_ok_cache", {})
        hit = cache.get(shape)
        if hit is not None:
            return hit
        m = self.m
        ok = m.head_start >= 1 and len(shape) == 4 and shape[1] == 3 and gops.stem_supported(shape[2], shape[3]) \
            and m.base.conv1.weight.shape[0] % 32 == 0
        if ok:
            h, w = shape[2] // 2, shape[3] // 2
            h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1                       # 3x3 / 2 max-pool
            for i in range(1, m.head_start):
                for u in getattr(m.base, f"layer{i}"):
                    convs = [u.conv1, u.conv2] + ([u.conv3] if u.kind != "basic" else [])
                    if u.downsample is not None:
                        c = u.downsample[0]
                        ok = ok and self._fits(h, w, c)
                    for c in convs:
                        ok = ok and self._fits(h, w, c)
                        k, st = c.kernel_size[0], c.stride[0]
                        h, w = (h + 2 * (k // 2) - k) // st + 1, (w + 2 * (k // 2) - k) // st + 1
        cache[shape] = bool(ok)
        return bool(ok)

    @staticmethod
    def _fits(h: int, w: int, conv: nn.Conv2d) -> bool:
        k, st, cin = conv.kernel_size[0], conv.stride[0], conv.in_channels
        if k == 1 and st == 1:
            return cin % 8 == 0
        return gops.conv_supported(h, w, cin, k, st)

    def _stem(self, x: torch.Tensor) -> torch.Tensor:
        """``x``: [B,3,H,W] (any memory format / float dtype) -> [B,H/4,W/4,64] bf16 NHWC."""
        base = self.m.base
        w = base.conv1.weight
        hit = self._stem_cache
        if hit is None or hit[0] != w._version or hit[1] != w.data_ptr():
            with torch.no_grad():
                w4 = gops.stem_weight_s2d(w.detach().float()).to(torch.bfloat16).contiguous()
            hit = self._stem_cache = (w._version, w.data_ptr(), w4)
        xn = x.permute(0, 2, 3, 1).to(torch.bfloat16).contiguous()
        b, h, wd, _ = xn.shape
        bn = base.bn1
        if bn.training:
            part = gops.col_part_buffer(b * (h // 2) * (wd // 2), w.shape[0], x.device)
            y = gops.stem_conv(xn, hit[2], None, relu=False, col_part=part)
            y = self._bn(y, bn, True, None, part)
        else:
            y = self._bn(gops.stem_conv(xn, hit[2], None, relu=False), bn, True)
        return gops.maxpool3x3s2(y)

    @torch.no_grad()
    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        m = self.m
        y = self._stem(x)
        for i in range(1, m.head_start):
            for u in getattr(m.base, f"layer{i}"):
                y = self._unit(y, u)
        return y.permute(0, 3, 1, 2)                     # logical NCHW over channels_last storage

    def batch_norms(self):
        m = self.m
        out = [m.base.bn1] if m.head_start >= 1 else []
        out += [b for i in range(1, m.head_start) for b in getattr(m.base, f"layer{i}").modules()
                if isinstance(b, nn.BatchNorm2d)]
        return out


def _make(name: str):
    def ctor(**kwargs):
        return ResNetReID(model_name=name, **kwargs)
    ctor.__name__ = name
    return ctor


resnet18, resnet34, resnet50, resnet101, resnet152 = (_make(n) for n in _SPECS)

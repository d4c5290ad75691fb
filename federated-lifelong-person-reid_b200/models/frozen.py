"""Inference-only execution of the frozen ResNet trunk (stem + ``layer1..k-1``) for FedSTIL's prototype pass
(``methods/fedstil.py:558-617``: eval-mode forward of the whole frozen trunk, repeated every epoch of every round).

What changes versus running the ``nn.Module``: batch-norm is folded into the preceding convolution once
(eval mode makes it an affine map), weights are kept as bf16 ``channels_last`` tensors, conv+bias+ReLU and
conv+bias+residual+ReLU are single fused calls, and a whole trunk pass for a given batch size is captured in a CUDA
graph so that ~160 module dispatches per batch collapse into one launch.

Execution paths of the residual stages (``native`` flag):
* **native** (default on CUDA when the shapes fit): every 1x1 convolution is a wgmma GEMM and every 3x3 / strided
  convolution an implicit GEMM of ``csrc/gemm_wgmma.cu`` (NHWC bf16, folded-BN bias + residual + ReLU in the lean
  epilogue, stride 2 through TMA element strides) - the same kernels as the trainable head;
* **library** fallback (cuDNN fused conv calls) for shapes the implicit-GEMM tiling does not cover.
The 7x7 / 2 stem (3 input channels) runs natively as a 4x4 convolution over 2x2 space-to-depth cells
(``ops.gemm.stem_conv``) followed by the NHWC max-pool kernel; ``FLPR_NATIVE_STEM=0`` keeps cuDNN / ATen for the two.
"""
from __future__ import annotations

import os
import threading
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F


def _fold(conv: nn.Conv2d, bn: nn.BatchNorm2d, dtype: torch.dtype) -> Tuple[torch.Tensor, torch.Tensor]:
    with torch.no_grad():
        scale = bn.weight.float() * torch.rsqrt(bn.running_var.float() + bn.eps)
        w = conv.weight.float() * scale.view(-1, 1, 1, 1)
        b = bn.bias.float() - bn.running_mean.float() * scale
        if conv.bias is not None:
            b = b + conv.bias.float() * scale
    return w.to(dtype).contiguous(memory_format=torch.channels_last), b.to(dtype).contiguous()


class FoldedTrunk:
    def __init__(self, net, dtype: torch.dtype = torch.bfloat16, use_graphs: bool = True):
        self.net = net
        self.dtype = dtype
        self.head_start = net.head_start
        self.device = next(net.parameters()).device
        self.ops: List[Tuple] = []
        base = net.base
        if self.head_start >= 1:
            w, b = _fold(base.conv1, base.bn1, dtype)
            self.ops.append(("conv_relu", w, b, base.conv1.stride, base.conv1.padding))
            self.ops.append(("maxpool",))
            for i in range(1, self.head_start):
                for u in getattr(base, f"layer{i}"):
                    self.ops.append(("unit", self._fold_unit(u)))
        self.use_graphs = use_graphs and self.device.type == "cuda"
        self._graphs: Dict[Tuple, List[dict]] = {}
        self._slot_lock = threading.Lock()
        self._fused_ok = self._probe_fused()
        self.native = True
        self._native_cache: Dict[Tuple, bool] = {}
        self._prepare_native()

    def _fold_unit(self, u) -> dict:
        d = {"kind": u.kind}
        d["c1"] = _fold(u.conv1, u.bn1, self.dtype) + (u.conv1.stride, u.conv1.padding)
        d["c2"] = _fold(u.conv2, u.bn2, self.dtype) + (u.conv2.stride, u.conv2.padding)
        if u.kind != "basic":
            d["c3"] = _fold(u.conv3, u.bn3, self.dtype) + (u.conv3.stride, u.conv3.padding)
        if u.downsample is not None:
            d["ds"] = _fold(u.downsample[0], u.downsample[1], self.dtype) + (u.downsample[0].stride,
                                                                              u.downsample[0].padding)
        return d

    def _probe_fused(self) -> bool:
        if self.device.type != "cuda":
            return False
        try:
            x = torch.zeros(1, 64, 8, 8, device=self.device, dtype=self.dtype).contiguous(
                memory_format=torch.channels_last)
            w = torch.zeros(64, 64, 3, 3, device=self.device, dtype=self.dtype).contiguous(
                memory_format=torch.channels_last)
            b = torch.zeros(64, device=self.device, dtype=self.dtype)
            torch.cudnn_convolution_relu(x, w, b, (1, 1), (1, 1), (1, 1), 1)
            torch.cudnn_convolution_add_relu(x, w, x, 1.0, b, (1, 1), (1, 1), (1, 1), 1)
            return True
        except Exception:
            return False

    # ------------------------------------------------------------------ functional forward
    def _conv(self, x, w, b, stride, padding, relu: bool, residual: Optional[torch.Tensor] = None):
        if self._fused_ok and relu:
            if residual is not None:
                return torch.cudnn_convolution_add_relu(x, w, residual, 1.0, b, stride, padding, (1, 1), 1)
            return torch.cudnn_convolution_relu(x, w, b, stride, padding, (1, 1), 1)
        y = F.conv2d(x, w, b, stride, padding)
        if residual is not None:
            y = y + residual
        return F.relu_(y) if relu else y

    # ------------------------------------------------------------------ native (wgmma) residual stages
    def _prepare_native(self) -> None:
        """OHWI bf16 weights + fp32 biases for the implicit-GEMM kernels."""
        from ..ops.gemm import stem_weight_s2d
        self._stem_w4 = self._stem_bias = None
        for op in self.ops:
            if op[0] == "conv_relu" and tuple(op[1].shape[1:]) == (3, 7, 7) and op[1].shape[0] % 32 == 0 \
                    and tuple(op[3]) == (2, 2) and tuple(op[4]) == (3, 3):
                self._stem_w4 = stem_weight_s2d(op[1].float()).to(self.dtype).contiguous()
                self._stem_bias = op[2].float().contiguous()
        for op in self.ops:
            if op[0] != "unit":
                continue
            d = op[1]
            for key in ("c1", "c2", "c3", "ds"):
                if key in d:
                    w, b, stride, padding = d[key]
                    d[key + "n"] = (w.permute(0, 2, 3, 1).contiguous(), b.float().contiguous(), int(stride[0]),
                                    int(padding[0]))

    def _native_ok(self, shape) -> bool:
        """Dry shape walk of :meth:`_forward_native`: every convolution must fit the implicit-GEMM tiling."""
        cached = self._native_cache.get(shape)
        if cached is not None:
            return cached
        from ..ops.gemm import conv_supported
        ok = getattr(self, "native", True) and self.device.type == "cuda" and self.dtype == torch.bfloat16

        def step(h, w, conv):
            wt, _, stride, padding = conv
            k, cin = wt.shape[1], wt.shape[3]
            good = (cin % 8 == 0) if (k == 1 and stride == 1) else conv_supported(h, w, cin, k, stride, padding)
            return good, (h + 2 * padding - k) // stride + 1, (w + 2 * padding - k) // stride + 1

        if ok:
            _, _, h, w = shape
            h, w = (h + 2 * 3 - 7) // 2 + 1, (w + 2 * 3 - 7) // 2 + 1         # 7x7 / 2 stem
            h, w = (h + 2 - 3) // 2 + 1, (w + 2 - 3) // 2 + 1                 # 3x3 / 2 max-pool
            for op in self.ops:
                if op[0] != "unit" or not ok:
                    continue
                d = op[1]
                if "dsn" in d:
                    ok = ok and step(h, w, d["dsn"])[0]
                g, h1, w1 = step(h, w, d["c1n"])
                ok = ok and g
                g, h1, w1 = step(h1, w1, d["c2n"])
                ok = ok and g
                if "c3n" in d:
                    g, h1, w1 = step(h1, w1, d["c3n"])
                    ok = ok and g
                h, w = h1, w1
        self._native_cache[shape] = bool(ok)
        return bool(ok)

    @staticmethod
    def _nconv(x: torch.Tensor, wt, b, stride: int, padding: int, relu: bool,
               residual: Optional[torch.Tensor] = None) -> torch.Tensor:
        """x: [N,H,W,C] bf16 contiguous -> [N,Ho,Wo,Cout]"""
        from ..ops import gemm as gops
        cout, k = wt.shape[0], wt.shape[1]
        n, h, w, c = x.shape
        if k == 1 and stride == 1:
            res2 = residual.reshape(-1, cout) if residual is not None else None
            y = gops.gemm(x.reshape(-1, c), wt.reshape(cout, c), bias_n=b, relu=relu, residual=res2)
            return y.view(n, h, w, cout)
        return gops.conv_nhwc(x, wt, padding=padding, stride=stride, bias=b, relu=relu, residual=residual)

    def _forward_native(self, x: torch.Tensor) -> torch.Tensor:
        from ..ops import gemm as gops
        native_stem = getattr(self, "native_stem", True) and os.environ.get("FLPR_NATIVE_STEM", "1") != "0" \
            and gops.stem_supported(x.shape[2], x.shape[3]) \
            and self._stem_w4 is not None
        for op in self.ops:
            if op[0] == "conv_relu":
                if native_stem:
                    # 7x7 / 2 stem as a 4x4 conv over space-to-depth cells on the wgmma kernel (NHWC in, NHWC out)
                    x = gops.stem_conv(x.permute(0, 2, 3, 1).contiguous(), self._stem_w4, self._stem_bias, relu=True)
                else:
                    x = self._conv(x, op[1], op[2], op[3], op[4], True)
            elif op[0] == "maxpool":
                if native_stem:
                    x = gops.maxpool3x3s2(x)
                else:
                    x = F.max_pool2d(x, 3, 2, 1)
                    x = x.permute(0, 2, 3, 1).contiguous()               # NHWC from here on (free for channels_last)
            else:
                d = op[1]
                identity = x if "dsn" not in d else self._nconv(x, *d["dsn"], relu=False)
                out = self._nconv(x, *d["c1n"], relu=True)
                if d["kind"] == "basic":
                    x = self._nconv(out, *d["c2n"], relu=True, residual=identity)
                else:
                    out = self._nconv(out, *d["c2n"], relu=True)
                    x = self._nconv(out, *d["c3n"], relu=True, residual=identity)
        return x.permute(0, 3, 1, 2)                                      # logical NCHW, channels_last memory

    def _forward(self, x: torch.Tensor) -> torch.Tensor:
        if self._native_ok(tuple(x.shape)) and any(op[0] == "unit" for op in self.ops):
            return self._forward_native(x)
        return self._forward_library(x)

    def _forward_library(self, x: torch.Tensor) -> torch.Tensor:
        for op in self.ops:
            if op[0] == "conv_relu":
                x = self._conv(x, op[1], op[2], op[3], op[4], True)
            elif op[0] == "maxpool":
                x = F.max_pool2d(x, 3, 2, 1)
            else:
                d = op[1]
                identity = x if "ds" not in d else self._conv(x, *d["ds"], relu=False)
                out = self._conv(x, *d["c1"], relu=True)
                if d["kind"] == "basic":
                    x = self._conv(out, *d["c2"], relu=True, residual=identity)
                else:
                    out = self._conv(out, *d["c2"], relu=True)
                    x = self._conv(out, *d["c3"], relu=True, residual=identity)
        return x

    @torch.no_grad()
    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        """``x``: float / bf16 ``[B,3,H,W]`` (any memory format). Returns the feature map at the cut (bf16,
        channels_last) as a tensor owned by the caller.

        One captured graph (+ static input / output buffers) per *slot* and batch shape. Concurrent callers (client
        threads on different streams) take different slots; a slot is handed over with an event so that its static
        buffers are never rewritten while a previous user's replay or read-out is still in flight."""
        x = x.to(self.dtype).contiguous(memory_format=torch.channels_last)
        if not self.use_graphs:
            return self._forward(x)
        key = tuple(x.shape)
        slot = self._acquire(key, x)
        try:
            cur = torch.cuda.current_stream(self.device)
            if slot["event"] is not None:
                cur.wait_event(slot["event"])
            slot["in"].copy_(x)
            slot["graph"].replay()
            out = slot["out"].clone()
            ev = torch.cuda.Event()
            ev.record(cur)
            slot["event"] = ev
        finally:
            with self._slot_lock:
                slot["busy"] = False
        return out

    def _acquire(self, key, x: torch.Tensor) -> dict:
        from ..runtime.graphs import CAPTURE_LOCK, capture
        with self._slot_lock:
            slots = self._graphs.setdefault(key, [])
            for sl in slots:
                if not sl["busy"]:
                    sl["busy"] = True
                    return sl
            sl = {"busy": True, "event": None, "graph": None}
            slots.append(sl)
        with CAPTURE_LOCK:
            static_in = x.clone()
            from ..ops import native
            side = native.dedicated_stream(self.device)
            side.wait_stream(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(side):
                for _ in range(2):
                    self._forward(static_in)
            torch.cuda.current_stream(self.device).wait_stream(side)
            g = torch.cuda.CUDAGraph()
            with capture(g):
                static_out = self._forward(static_in)
            sl["graph"], sl["in"], sl["out"] = g, static_in, static_out
        return sl


_SHARED: Dict[Tuple, FoldedTrunk] = {}


def shared_folded_trunk(net, dtype: torch.dtype = torch.bfloat16) -> FoldedTrunk:
    """One folded trunk per (architecture, device) is shared by all clients of a rank whose frozen weights are equal
    (FedSTIL never changes the trunk; all clients start from the same pre-trained weights)."""
    dev = next(net.parameters()).device
    key = (net.model_name, str(dev), net.head_start, dtype)
    ft = _SHARED.get(key)
    if ft is not None:
        a, b = ft.net.base.conv1.weight, net.base.conv1.weight
        la, lb = getattr(ft.net.base, "layer1")[0].conv1.weight, getattr(net.base, "layer1")[0].conv1.weight
        if a.shape == b.shape and torch.equal(a, b) and torch.equal(la, lb) and \
                torch.equal(ft.net.base.bn1.running_var, net.base.bn1.running_var):
            return ft
        return FoldedTrunk(net, dtype)
    ft = FoldedTrunk(net, dtype)
    _SHARED[key] = ft
    return ft

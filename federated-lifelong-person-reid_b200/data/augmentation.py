"""Augmentation registry with the reference's five levels (``datasets/image_augmentation.py:6-71``).

Two implementations per level:
* ``host_transform``   – torchvision ``Compose`` identical in op order to the reference
  (ToTensor -> Normalize -> [HFlip -> RandomErasing(p)] -> Resize), used by the per-sample DataLoader path.
* ``DeviceAugment``    – the same pipeline applied to a whole uint8 NHWC batch on the GPU (normalise, flip, erase)
  after a one-time resize at task-load time; this is what the engine uses by default.
"""
from __future__ import annotations

import math
from typing import Dict, Sequence

import torch

ERASE_P: Dict[str, float] = {"none": 0.0, "default": 0.5, "rose": 0.6, "sharp": 0.75, "drastic": 0.9}
FLIP_P: Dict[str, float] = {"none": 0.0, "default": 0.5, "rose": 0.5, "sharp": 0.5, "drastic": 0.5}


def host_transform(level: str, size: Sequence[int] = (384, 128), mean=(0.485, 0.456, 0.406),
                   std=(0.229, 0.224, 0.225)):
    import torchvision.transforms as T
    ops = [T.ToTensor(), T.Normalize(mean, std)]
    if level != "none":
        ops += [T.RandomHorizontalFlip(p=FLIP_P[level]), T.RandomErasing(p=ERASE_P[level])]
    ops.append(T.Resize(list(size)))
    return T.Compose(ops)


def _factory(level: str):
    def make(size=(384, 128), mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225)):
        return host_transform(level, size, mean, std)
    make.__name__ = f"augmentation_{level}"
    return make


augmentations = {lvl: _factory(lvl) for lvl in ERASE_P}


class DeviceAugment:
    """Batched GPU augmentation: uint8 ``[B,H,W,3]`` -> normalised float ``[B,3,H,W]`` (channels_last memory)."""

    def __init__(self, level: str, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225),
                 dtype: torch.dtype = torch.float32, scale=(0.02, 0.33), ratio=(0.3, 3.3)):
        self.level = level
        self.mean = torch.tensor(mean, dtype=torch.float32).view(1, 1, 1, 3) * 255.0
        self.inv_std = 1.0 / (torch.tensor(std, dtype=torch.float32).view(1, 1, 1, 3) * 255.0)
        self.mean01 = torch.tensor(mean, dtype=torch.float32).view(1, 1, 1, 3)
        self.std = torch.tensor(std, dtype=torch.float32).view(1, 1, 1, 3)
        self.dtype = dtype
        self.scale, self.ratio = scale, ratio

    def _native(self, u8: torch.Tensor, generator) -> torch.Tensor:
        """One fused sm_90a kernel (``csrc/fused_ops.cu: augment_u8_kernel``): normalise + flip + erase + cast."""
        import ctypes as C
        from ..ops import native
        lib = native.kernels()
        b, h, w, _ = u8.shape
        u8 = u8.contiguous()
        u = torch.rand(7, b, device=u8.device, generator=generator)
        out = torch.empty(b, h, w, 3, dtype=self.dtype, device=u8.device)
        if getattr(self, "_consts", None) is None:
            m = self.mean.flatten().tolist()
            i = self.inv_std.flatten().tolist()
            self._consts = ((C.c_float * 3)(*m), (C.c_float * 3)(*i))
        mean3, inv3 = self._consts
        rc = lib.flpr_augment_u8(native.ptr(u8), native.ptr(out), native.ptr(u), b, h, w,
                                 C.cast(mean3, C.c_void_p), C.cast(inv3, C.c_void_p),
                                 FLIP_P[self.level], ERASE_P[self.level], self.scale[0], self.scale[1],
                                 self.ratio[0], self.ratio[1], int(self.dtype == torch.bfloat16),
                                 native.stream_of(u8.device))
        native.check(rc, "flpr_augment_u8")
        native.count_launch()
        return out.permute(0, 3, 1, 2)

    def __call__(self, u8: torch.Tensor, generator: torch.Generator | None = None) -> torch.Tensor:
        from ..ops import native
        if native.on_device(u8, "flpr_augment_u8") and u8.shape[2] % 4 == 0 \
                and self.dtype in (torch.bfloat16, torch.float32) and u8.dtype == torch.uint8:
            return self._native(u8, generator)
        return self.reference(u8, generator)

    def reference(self, u8: torch.Tensor, generator: torch.Generator | None = None) -> torch.Tensor:
        """Plain tensor-op implementation (CPU path and numerics reference of the fused kernel); consumes the same
        ``[7, B]`` block of uniforms as the kernel, so both produce the same batch from the same generator state."""
        dev = u8.device
        if self.mean.device != dev:
            self.mean, self.inv_std = self.mean.to(dev), self.inv_std.to(dev)
        if dev.type == "cpu":
            # the rounding sequence of torchvision's ToTensor + Normalize (image_augmentation.py:6-71): the fp32 CPU
            # path then feeds the network bit-identical inputs to the reference's
            x = (u8.float().div_(255.0) - self.mean01) / self.std          # [B,H,W,3]
        else:
            x = (u8.float() - self.mean) * self.inv_std                       # [B,H,W,3]
        b, h, w, _ = x.shape
        u = torch.rand(7, b, device=dev, generator=generator)
        if self.level != "none":
            flip = u[0] < FLIP_P[self.level]
            x = torch.where(flip.view(b, 1, 1, 1), x.flip(2), x)
            # RandomErasing(value=0): one rectangle per selected sample, area in `scale`, aspect log-uniform in `ratio`
            sel = u[1] < ERASE_P[self.level]
            area = (u[2] * (self.scale[1] - self.scale[0]) + self.scale[0]) * h * w
            logr = u[3] * (math.log(self.ratio[1]) - math.log(self.ratio[0])) + math.log(self.ratio[0])
            ar = torch.exp(logr)
            eh = torch.sqrt(area * ar).round().clamp(1, h - 1)
            ew = torch.sqrt(area / ar).round().clamp(1, w - 1)
            top = (u[4] * (h - eh + 1)).floor()
            left = (u[5] * (w - ew + 1)).floor()
            ys = torch.arange(h, device=dev).view(1, h, 1)
            xs = torch.arange(w, device=dev).view(1, 1, w)
            box = (ys >= top.view(b, 1, 1)) & (ys < (top + eh).view(b, 1, 1)) & \
                  (xs >= left.view(b, 1, 1)) & (xs < (left + ew).view(b, 1, 1)) & sel.view(b, 1, 1)
            x = x.masked_fill(box.unsqueeze(-1), 0.0)
        # logical NCHW view over NHWC storage == torch.channels_last (CUDA); plain contiguous NCHW on the CPU
        out = x.to(self.dtype).permute(0, 3, 1, 2)
        return out if dev.type == "cuda" else out.contiguous()

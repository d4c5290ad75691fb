"""Swin-Transformer ReID backbones (tiny / small / base / large) – capability parity with
``models/swin_transformer.py`` of the reference (timm-derived): shifted-window attention with relative position
bias, patch merging, stochastic depth, optional activation checkpointing, 224x224 bilinear resize inside
``forward``, BNNeck + classifier head, train -> ``(cls_score, global_feat)`` / eval -> ``global_feat``.
Parameter names follow timm's (``base.patch_embed.proj``, ``base.layers.{i}.blocks.{j}.attn.qkv`` ...), so
``fine_tuning: [base.layers.3, classifier]`` and reference checkpoints address the same tensors.

Written from the architecture description, not from the reference source. H100-first choices: the attention core is
one fused ``scaled_dot_product_attention`` call per block with the relative-position bias and the shift mask merged
into a single additive bias tensor that is cached per (window grid, shift); window (un)partition is a pure reshape /
permute pair; the network exposes the same *frozen trunk | trainable head* split as the ResNets
(``configure_split`` / ``forward_trunk`` / ``forward_head``) so FedSTIL prototypes are the 49x768 token maps entering
``layers.3``.
"""
from __future__ import annotations

import os
from typing import Optional, Sequence, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F
import torch.utils.checkpoint as ckpt

_SPECS = {
    "swin_tiny": dict(embed_dim=96, depths=(2, 2, 6, 2), num_heads=(3, 6, 12, 24)),
    "swin_small": dict(embed_dim=96, depths=(2, 2, 18, 2), num_heads=(3, 6, 12, 24)),
    "swin_base": dict(embed_dim=128, depths=(2, 2, 18, 2), num_heads=(4, 8, 16, 32)),
    "swin_large": dict(embed_dim=192, depths=(2, 2, 18, 2), num_heads=(6, 12, 24, 48)),
}


from ..ops import layer as lops  # noqa: E402


class TcLinear(nn.Linear):
    """``nn.Linear`` whose CUDA / bf16 forward, data gradient and weight gradient run on the wgmma GEMM kernel
    (``ops.gemm.linear``: bf16 compute copy of the weight kept by the fused optimizer, fp32 weight gradient written by
    the GEMM epilogue straight into the parameter's slot of the arena gradient buffer). Same parameters, same
    ``state_dict`` keys: an existing ``nn.Linear`` is switched over by re-classing it (:func:`use_tensor_core_linears`).
    The bias stays an fp32 parameter; its gradient is the column sum of the output gradient (autograd)."""

    _flpr_shadow = None          # param -> bf16 view (ParamArena.shadow_of)
    _flpr_grad_slot = None       # param -> fp32 gradient view (ParamArena.grad_of)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        w = self.weight
        native_ok = x.is_cuda and w.shape[0] % 8 == 0 and w.shape[1] % 8 == 0 and (
            x.dtype == torch.bfloat16 or (x.dtype == torch.float32 and torch.is_autocast_enabled()))
        if not native_ok:
            return F.linear(x, w.to(x.dtype) if w.dtype != x.dtype else w,
                            None if self.bias is None else self.bias.to(x.dtype))
        from ..ops import gemm as gops
        sh = self._flpr_shadow(w) if self._flpr_shadow is not None else None
        if sh is None and not w.requires_grad:
            sh = self._frozen_copy(w)                          # frozen stage: cached bf16 copy
        gs = self._flpr_grad_slot(w) if (self._flpr_grad_slot is not None and w.requires_grad) else None
        x2 = x.reshape(-1, x.shape[-1])
        y = gops.linear(x2 if x2.dtype == torch.bfloat16 else x2.to(torch.bfloat16), w, sh, gs, False, self.bias)
        return y.view(*x.shape[:-1], w.shape[0])

    def _frozen_copy(self, w: torch.Tensor) -> torch.Tensor:
        hit = self.__dict__.get("_flpr_wb")
        if hit is None or hit[0] != w._version or hit[1] != w.data_ptr():
            hit = self.__dict__["_flpr_wb"] = (w._version, w.data_ptr(), w.detach().to(torch.bfloat16))
        return hit[2]


class FrozenLayerNorm(nn.LayerNorm):
    """LayerNorm of a FROZEN stage on the bf16 path: under autocast ``layer_norm`` is an fp32 op, which turns the whole
    residual stream of the inference-only trunk into fp32 (twice the HBM traffic for every add / norm / cast). With
    frozen parameters and no gradient the bf16 kernel (fp32 statistics inside) is used on bf16 activations instead."""

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if not (x.is_cuda and x.dtype == torch.bfloat16 and not torch.is_grad_enabled()
                and not self.weight.requires_grad):
            return super().forward(x)
        hit = self.__dict__.get("_flpr_wb")
        w = self.weight
        if hit is None or hit[0] != (w._version, self.bias._version):
            hit = self.__dict__["_flpr_wb"] = ((w._version, self.bias._version), w.detach().to(torch.bfloat16),
                                               self.bias.detach().to(torch.bfloat16))
        c = x.shape[-1]
        if c % 8 == 0 and c <= 2048 and len(self.normalized_shape) == 1 and w.dtype == torch.float32 \
                and self.bias is not None and lops.enabled("swin_tokens", x.device):
            # native warp-per-token kernel (fp32 statistics, fp32 gamma / beta): one pass over the tokens where ATen's
            # bf16 LayerNorm takes several
            x2 = x.reshape(-1, c)
            return lops.ln_rows(x2 if x2.is_contiguous() else x2.contiguous(), self.weight, self.bias,
                                self.eps).view(x.shape)
        with torch.autocast(device_type="cuda", enabled=False):
            return F.layer_norm(x, self.normalized_shape, hit[1], hit[2], self.eps)


class TrainLayerNorm(nn.LayerNorm):
    """``norm1`` / ``norm2`` of a TRAINABLE Swin block on the bf16 path (``models/swin_transformer.py:358-395``): the
    native warp-per-token kernels (``ops.layer.layer_norm_rows``: fp32 statistics, fp32 ``gamma`` / ``beta``, bf16 in and
    out, one-sweep backward with deterministic ``dgamma`` / ``dbeta``) instead of the autocast ``layer_norm`` (an fp32 op:
    fp32 output + a cast pass in front of the tensor-core Linear that consumes it, and the mirror image in backward).
    Only block norms are switched - their consumer casts to bf16 anyway, so the GEMM operands are unchanged; the final
    ``norm`` in front of the pooled feature stays fp32."""

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        c = x.shape[-1]
        if not (x.is_cuda and x.dtype == torch.bfloat16 and torch.is_grad_enabled() and self.weight.requires_grad
                and len(self.normalized_shape) == 1 and c % 8 == 0 and c <= 2048 and self.bias is not None
                and self.weight.dtype == torch.float32 and self.weight.data_ptr() % 16 == 0
                and self.bias.data_ptr() % 16 == 0 and lops.enabled("ln_train", x.device)):
            return super().forward(x)
        x2 = x.reshape(-1, c)
        y = lops.layer_norm_rows(x2 if x2.is_contiguous() else x2.contiguous(), self.weight, self.bias, self.eps)
        return y.view(x.shape)


def use_tensor_core_linears(root: nn.Module, shadow=None, grad_slot=None) -> int:
    """Re-class every plain ``nn.Linear`` under ``root`` to :class:`TcLinear` (and the frozen ``nn.LayerNorm``s to
    :class:`FrozenLayerNorm`); returns how many Linears were switched."""
    n = 0
    for m in root.modules():
        if type(m) is nn.Linear:
            m.__class__ = TcLinear
            m._flpr_shadow, m._flpr_grad_slot = shadow, grad_slot
            n += 1
        elif type(m) is nn.LayerNorm and m.elementwise_affine and not m.weight.requires_grad:
            m.__class__ = FrozenLayerNorm
    for blk in root.modules():
        if isinstance(blk, SwinTransformerBlock):
            for ln in (blk.norm1, blk.norm2):
                if type(ln) is nn.LayerNorm and ln.elementwise_affine and ln.weight.requires_grad:
                    ln.__class__ = TrainLayerNorm
    return n


class DropPath(nn.Module):
    def __init__(self, p: float = 0.0):
        super().__init__()
        self.p = float(p)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if self.p == 0.0 or not self.training:
            return x
        keep = 1.0 - self.p
        mask = x.new_empty((x.shape[0],) + (1,) * (x.dim() - 1)).bernoulli_(keep)
        return x * mask / keep


class Mlp(nn.Module):
    def __init__(self, dim: int, hidden: int, drop: float = 0.0):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.act = nn.GELU()
        self.fc2 = nn.Linear(hidden, dim)
        self.drop = nn.Dropout(drop)

    def forward(self, x):
        h = self.fc1(x)
        if h.is_cuda and h.dtype == torch.bfloat16 and torch.is_grad_enabled() and h.requires_grad \
                and h.numel() % 8 == 0 and lops.enabled("ln_train", h.device) and lops.enabled("swin_tokens", h.device):
            h = lops.gelu_act(h if h.is_contiguous() else h.contiguous())   # native forward / backward (trainable stage)
        else:
            h = self.act(h)
        return self.drop(self.fc2(self.drop(h)))


def window_partition(x: torch.Tensor, ws: int) -> torch.Tensor:
    """[B,H,W,C] -> [B*nW, ws*ws, C]"""
    b, h, w, c = x.shape
    x = x.view(b, h // ws, ws, w // ws, ws, c).permute(0, 1, 3, 2, 4, 5)
    return x.reshape(-1, ws * ws, c)


def window_reverse(win: torch.Tensor, ws: int, h: int, w: int) -> torch.Tensor:
    """[B*nW, ws*ws, C] -> [B,H,W,C]"""
    b = win.shape[0] // ((h // ws) * (w // ws))
    x = win.view(b, h // ws, w // ws, ws, ws, -1).permute(0, 1, 3, 2, 4, 5)
    return x.reshape(b, h, w, -1)


class WindowAttention(nn.Module):
    def __init__(self, dim: int, window_size: int, num_heads: int, qkv_bias: bool = True, attn_drop: float = 0.0,
                 proj_drop: float = 0.0):
        super().__init__()
        self.dim, self.ws, self.num_heads = dim, window_size, num_heads
        self.scale = (dim // num_heads) ** -0.5
        self.relative_position_bias_table = nn.Parameter(torch.zeros((2 * window_size - 1) ** 2, num_heads))
        coords = torch.stack(torch.meshgrid(torch.arange(window_size), torch.arange(window_size), indexing="ij"))
        flat = coords.flatten(1)
        rel = (flat[:, :, None] - flat[:, None, :]).permute(1, 2, 0).contiguous()
        rel[:, :, 0] += window_size - 1
        rel[:, :, 1] += window_size - 1
        rel[:, :, 0] *= 2 * window_size - 1
        self.register_buffer("relative_position_index", rel.sum(-1))
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.attn_drop = attn_drop
        self.proj = nn.Linear(dim, dim)
        self.proj_drop = nn.Dropout(proj_drop)
        nn.init.trunc_normal_(self.relative_position_bias_table, std=0.02)

    def bias(self, mask: Optional[torch.Tensor]) -> torch.Tensor:
        """Additive attention bias ``[nW or 1, heads, N, N]`` = relative position bias (+ shift mask)."""
        t = self.relative_position_bias_table
        frozen = not t.requires_grad and not torch.is_grad_enabled()
        if frozen:
            # frozen stage: the table only changes through in-place loads (dispatch, checkpoint restore), which bump
            # ``_version`` - the gathered / permuted (+ masked) bias is reused across forward passes
            key = (t._version, t.data_ptr(), None if mask is None else mask.data_ptr())
            hit = self.__dict__.get("_flpr_bias")
            if hit is not None and hit[0] == key:
                return hit[1]
        n = self.ws * self.ws
        b = t[self.relative_position_index.view(-1)].view(n, n, -1)
        b = b.permute(2, 0, 1).unsqueeze(0)
        if mask is not None:
            b = b + mask.unsqueeze(1)
        if frozen:
            b = b.contiguous()
            self.__dict__["_flpr_bias"] = (key, b)
        return b

    def forward(self, x: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        bw, n, c = x.shape
        qkv5 = self.qkv(x).view(bw, n, 3, self.num_heads, c // self.num_heads)
        drop = self.attn_drop if self.training else 0.0
        if drop == 0.0 and getattr(self, "fused", True):
            from ..ops.fused import window_attention, window_attention_supported
            if window_attention_supported(qkv5):
                # one fused kernel per (window, head): QK^T + bias (+ mask) -> softmax -> PV, scores never leave the SM
                out = window_attention(qkv5, self.bias(mask), self.scale)
                return self.proj_drop(self.proj(out))
        qkv = qkv5.permute(2, 0, 3, 1, 4)
        q, k, v = qkv[0], qkv[1], qkv[2]
        bias = self.bias(mask).to(q.dtype)
        if mask is not None:
            nw = mask.shape[0]
            q, k, v = (t.view(bw // nw, nw, self.num_heads, n, -1) for t in (q, k, v))
            out = F.scaled_dot_product_attention(q, k, v, attn_mask=bias.unsqueeze(0), dropout_p=drop, scale=self.scale)
            out = out.reshape(bw, self.num_heads, n, -1)
        else:
            out = F.scaled_dot_product_attention(q, k, v, attn_mask=bias, dropout_p=drop, scale=self.scale)
        return self.proj_drop(self.proj(out.transpose(1, 2).reshape(bw, n, c)))


class SwinTransformerBlock(nn.Module):
    def __init__(self, dim: int, resolution: Tuple[int, int], num_heads: int, window_size: int = 7, shift_size: int = 0,
                 mlp_ratio: float = 4.0, qkv_bias: bool = True, drop: float = 0.0, attn_drop: float = 0.0,
                 drop_path: float = 0.0):
        super().__init__()
        self.dim, self.resolution = dim, resolution
        self.window_size, self.shift_size = window_size, shift_size
        if min(resolution) <= window_size:
            self.shift_size, self.window_size = 0, min(resolution)
        assert 0 <= self.shift_size < self.window_size, "shift_size must in 0-window_size"
        self.norm1 = nn.LayerNorm(dim)
        self.attn = WindowAttention(dim, self.window_size, num_heads, qkv_bias, attn_drop, drop)
        self.drop_path = DropPath(drop_path)
        self.norm2 = nn.LayerNorm(dim)
        self.mlp = Mlp(dim, int(dim * mlp_ratio), drop)
        mask = None
        if self.shift_size > 0:
            h, w = resolution
            img = torch.zeros(1, h, w, 1)
            cnt = 0
            spans = (slice(0, -self.window_size), slice(-self.window_size, -self.shift_size),
                     slice(-self.shift_size, None))
            for hs in spans:
                for ws_ in spans:
                    img[:, hs, ws_, :] = cnt
                    cnt += 1
            mw = window_partition(img, self.window_size).squeeze(-1)
            mask = mw.unsqueeze(1) - mw.unsqueeze(2)
            mask = mask.masked_fill(mask != 0, -100.0).masked_fill(mask == 0, 0.0)
        self.register_buffer("attn_mask", mask)

    def _fused_ok(self, x: torch.Tensor) -> bool:
        """Frozen stage on the bf16 inference path (prototype pass / frozen stages of a training step)."""
        if not (x.is_cuda and x.dtype == torch.bfloat16 and not torch.is_grad_enabled()):
            return False
        c = x.shape[-1]
        if c % 8 or c > 2048 or self.window_size * self.window_size < 1:
            return False
        if self.training and (self.drop_path.p > 0.0 or self.mlp.drop.p > 0.0):
            return False
        frozen = not any(p.requires_grad for p in (self.norm1.weight, self.norm2.weight, self.mlp.fc1.weight,
                                                   self.mlp.fc2.weight))
        fp32 = all(p is not None and p.dtype == torch.float32 for p in (
            self.norm1.weight, self.norm1.bias, self.norm2.weight, self.norm2.bias, self.mlp.fc2.bias))
        return frozen and fp32 and lops.enabled("swin_tokens", x.device)

    def _forward_fused(self, x: torch.Tensor) -> torch.Tensor:
        """Same block, four fewer passes over the token stream: ``norm1`` writes straight into the layout of the shifted
        windows (norm + roll + window partition = one kernel), window reverse + roll back + residual is one kernel,
        ``norm2`` is the native LayerNorm, and the second residual add happens in the ``fc2`` GEMM epilogue."""
        from ..ops import gemm as gops
        h, w = self.resolution
        b, l, c = x.shape
        ws, sh = self.window_size, self.shift_size
        x2 = x.reshape(b * l, c)
        x2 = x2 if x2.is_contiguous() else x2.contiguous()
        win = lops.ln_rows(x2, self.norm1.weight, self.norm1.bias, self.norm1.eps, (h, w, ws, sh))
        win = self.attn(win.view(-1, ws * ws, c), self.attn_mask).reshape(-1, c)
        if win.dtype != torch.bfloat16:
            win = win.to(torch.bfloat16)
        x2 = lops.window_merge_add(win if win.is_contiguous() else win.contiguous(), x2, h, w, ws, sh)
        y = lops.ln_rows(x2, self.norm2.weight, self.norm2.bias, self.norm2.eps)
        hid = self.mlp.fc1(y).reshape(b * l, -1)
        hid = lops.gelu_rows(hid if (hid.dtype == torch.bfloat16 and hid.is_contiguous())
                             else hid.to(torch.bfloat16).contiguous())
        fc2 = self.mlp.fc2
        wb = fc2._frozen_copy(fc2.weight) if hasattr(fc2, "_frozen_copy") else fc2.weight.detach().to(torch.bfloat16)
        out = gops.gemm(hid, wb, bias_n=fc2.bias.detach().float(), residual=x2)
        return out.view(b, l, c)

    def _fused_train_ok(self, x: torch.Tensor) -> bool:
        """Trainable stage on the bf16 path: both block norms are :class:`TrainLayerNorm` (fp32 affine parameters in the
        arena) and the LayerNorm / merge kernels passed their self-check."""
        if not (x.is_cuda and x.dtype == torch.bfloat16 and torch.is_grad_enabled()):
            return False
        c = x.shape[-1]
        if c % 8 or c > 2048 or type(self.norm1) is not TrainLayerNorm or type(self.norm2) is not TrainLayerNorm:
            return False
        for p in (self.norm1.weight, self.norm1.bias, self.norm2.weight, self.norm2.bias):
            if p is None or p.dtype != torch.float32 or p.data_ptr() % 16:
                return False
        return lops.enabled("ln_train", x.device)

    def _drop_scale(self, batch: int, like: torch.Tensor) -> Optional[torch.Tensor]:
        """This call's stochastic-depth factors ``[B]`` (0 or ``1 / keep``), drawn exactly like :class:`DropPath` does."""
        p = self.drop_path.p
        if p == 0.0 or not self.training:
            return None
        keep = 1.0 - p
        mask = like.new_empty((batch, 1, 1)).bernoulli_(keep)
        return (mask.float().view(batch) / keep).contiguous()

    def _forward_fused_train(self, x: torch.Tensor) -> torch.Tensor:
        """The trainable block with the token passes of the first half fused (``models/swin_transformer.py:358-395``):
        ``norm1`` writes straight into the layout of the shifted windows (norm + roll + window partition: one kernel
        forward, one backward), and window reverse + roll back + drop-path scaling + residual add is one kernel (its
        backward: one gather). ``norm2`` is the native LayerNorm; the MLP half keeps its module form."""
        h, w = self.resolution
        b, l, c = x.shape
        ws, sh = self.window_size, self.shift_size
        x2 = x.reshape(b * l, c)
        x2 = x2 if x2.is_contiguous() else x2.contiguous()
        win = lops.layer_norm_rows(x2, self.norm1.weight, self.norm1.bias, self.norm1.eps, (h, w, ws, sh))
        att = self.attn(win.view(-1, ws * ws, c), self.attn_mask).reshape(-1, c)
        if att.dtype != x2.dtype:
            att = att.to(x2.dtype)
        x2 = lops.window_merge_residual(att if att.is_contiguous() else att.contiguous(), x2, self._drop_scale(b, x2),
                                        h, w, ws, sh)
        x3 = x2.view(b, l, c)
        return x3 + self.drop_path(self.mlp(self.norm2(x3)))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        h, w = self.resolution
        b, l, c = x.shape
        assert l == h * w, "input feature has wrong size"
        if self._fused_ok(x):
            return self._forward_fused(x)
        if self._fused_train_ok(x):
            return self._forward_fused_train(x)
        shortcut = x
        x = self.norm1(x).view(b, h, w, c)
        if self.shift_size > 0:
            x = torch.roll(x, shifts=(-self.shift_size, -self.shift_size), dims=(1, 2))
        win = window_partition(x, self.window_size)
        win = self.attn(win, self.attn_mask)
        x = window_reverse(win, self.window_size, h, w)
        if self.shift_size > 0:
            x = torch.roll(x, shifts=(self.shift_size, self.shift_size), dims=(1, 2))
        x = shortcut + self.drop_path(x.view(b, l, c))
        return x + self.drop_path(self.mlp(self.norm2(x)))


class PatchMerging(nn.Module):
    def __init__(self, resolution: Tuple[int, int], dim: int):
        super().__init__()
        self.resolution, self.dim = resolution, dim
        self.reduction = nn.Linear(4 * dim, 2 * dim, bias=False)
        self.norm = nn.LayerNorm(4 * dim)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        h, w = self.resolution
        b, l, c = x.shape
        x = x.view(b, h // 2, 2, w // 2, 2, c).permute(0, 1, 3, 4, 2, 5).reshape(b, (h // 2) * (w // 2), 4 * c)
        return self.reduction(self.norm(x))


class BasicLayer(nn.Module):
    def __init__(self, dim, resolution, depth, num_heads, window_size, mlp_ratio, qkv_bias, drop, attn_drop, drop_path,
                 downsample: bool, use_checkpoint: bool):
        super().__init__()
        self.use_checkpoint = use_checkpoint
        self.blocks = nn.ModuleList([
            SwinTransformerBlock(dim, resolution, num_heads, window_size, 0 if i % 2 == 0 else window_size // 2,
                                 mlp_ratio, qkv_bias, drop, attn_drop, drop_path[i]) for i in range(depth)])
        self.downsample = PatchMerging(resolution, dim) if downsample else None

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        for blk in self.blocks:
            if self.use_checkpoint and self.training and torch.is_grad_enabled():
                x = ckpt.checkpoint(blk, x, use_reentrant=False)
            else:
                x = blk(x)
        return x if self.downsample is None else self.downsample(x)


class PatchEmbed(nn.Module):
    def __init__(self, img_size=224, patch_size=4, in_chans=3, embed_dim=96, norm: bool = True):
        super().__init__()
        self.img_size = (img_size, img_size)
        self.grid_size = (img_size // patch_size, img_size // patch_size)
        self.num_patches = self.grid_size[0] * self.grid_size[1]
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size)
        self.norm = nn.LayerNorm(embed_dim) if norm else nn.Identity()

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.norm(self.proj(x).flatten(2).transpose(1, 2))


class SwinTransformer(nn.Module):
    def __init__(self, img_size=224, patch_size=4, in_chans=3, num_classes=1000, embed_dim=96, depths=(2, 2, 6, 2),
                 num_heads=(3, 6, 12, 24), window_size=7, mlp_ratio=4.0, qkv_bias=True, drop_rate=0.0,
                 attn_drop_rate=0.0, drop_path_rate=0.1, ape=False, patch_norm=True, use_checkpoint=False):
        super().__init__()
        self.num_layers = len(depths)
        self.embed_dim = embed_dim
        self.num_features = int(embed_dim * 2 ** (self.num_layers - 1))
        self.patch_embed = PatchEmbed(img_size, patch_size, in_chans, embed_dim, patch_norm)
        self.patch_grid = self.patch_embed.grid_size
        self.absolute_pos_embed = None
        if ape:
            self.absolute_pos_embed = nn.Parameter(torch.zeros(1, self.patch_embed.num_patches, embed_dim))
            nn.init.trunc_normal_(self.absolute_pos_embed, std=0.02)
        self.pos_drop = nn.Dropout(drop_rate)
        dpr = torch.linspace(0, drop_path_rate, sum(depths)).tolist()
        layers = []
        for i, depth in enumerate(depths):
            res = (self.patch_grid[0] // (2 ** i), self.patch_grid[1] // (2 ** i))
            layers.append(BasicLayer(int(embed_dim * 2 ** i), res, depth, num_heads[i], window_size, mlp_ratio,
                                     qkv_bias, drop_rate, attn_drop_rate, dpr[sum(depths[:i]):sum(depths[:i + 1])],
                                     downsample=i < self.num_layers - 1, use_checkpoint=use_checkpoint))
        self.layers = nn.ModuleList(layers)
        self.norm = nn.LayerNorm(self.num_features)
        self.avgpool = nn.AdaptiveAvgPool1d(1)
        self.head = nn.Linear(self.num_features, num_classes) if num_classes > 0 else nn.Identity()
        self.apply(self._init)

    @staticmethod
    def _init(m: nn.Module) -> None:
        if isinstance(m, nn.Linear):
            nn.init.trunc_normal_(m.weight, std=0.02)
            if m.bias is not None:
                nn.init.zeros_(m.bias)
        elif isinstance(m, nn.LayerNorm):
            nn.init.ones_(m.weight)
            nn.init.zeros_(m.bias)

    def embed(self, x: torch.Tensor) -> torch.Tensor:
        x = self.patch_embed(x)
        if self.absolute_pos_embed is not None:
            x = x + self.absolute_pos_embed
        return self.pos_drop(x)

    def run_layers(self, x: torch.Tensor, start: int, stop: int) -> torch.Tensor:
        for i in range(start, stop):
            x = self.layers[i](x)
        return x

    def pool(self, x: torch.Tensor) -> torch.Tensor:
        return self.avgpool(self.norm(x).transpose(1, 2)).flatten(1)

    def forward_features(self, x: torch.Tensor) -> torch.Tensor:
        return self.pool(self.run_layers(self.embed(x), 0, self.num_layers))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.head(self.forward_features(x))


class SwinTransformerReID(nn.Module):
    def __init__(self, model_name: str, num_classes: int = 1000, neck: str = "no",
                 pretrained_path: Optional[str] = None, **kwargs):
        super().__init__()
        swin_kw = {k: kwargs.pop(k) for k in ("drop_path_rate", "use_checkpoint", "ape") if k in kwargs}
        for k, v in kwargs.items():
            setattr(self, k, v)
        if model_name not in _SPECS:
            raise ValueError(f"No model named {model_name} for generating.")
        self.model_name, self.num_classes, self.neck = model_name, num_classes, neck
        self.base = SwinTransformer(patch_size=4, window_size=7, **_SPECS[model_name], **swin_kw)
        if pretrained_path and os.path.exists(pretrained_path):
            sd = torch.load(pretrained_path, map_location="cpu")
            self.base.load_state_dict(sd.get("model", sd), strict=False)
        self.in_planes = self.base.head.in_features
        self.base.head = nn.Sequential()
        if neck == "no":
            self.classifier = nn.Linear(self.in_planes, num_classes)
        elif neck == "bnneck":
            self.bottleneck = nn.BatchNorm1d(self.in_planes)
            self.bottleneck.bias.requires_grad_(False)
            self.classifier = nn.Linear(self.in_planes, num_classes, bias=False)
            nn.init.ones_(self.bottleneck.weight)
            nn.init.zeros_(self.bottleneck.bias)
            nn.init.normal_(self.classifier.weight, std=0.001)
        else:
            raise ValueError(f"Mismatched neck type for {neck}.")
        self.head_start = self.base.num_layers

    def configure_split(self, fine_tuning: Optional[Sequence[str]]) -> int:
        start = self.base.num_layers
        if not fine_tuning:
            start = 0
        else:
            for name in fine_tuning:
                if name == "base" or name.startswith("base.patch_embed") or name.startswith("base.absolute_pos_embed"):
                    start = 0
                for i in range(self.base.num_layers):
                    if name == f"base.layers.{i}" or name.startswith(f"base.layers.{i}."):
                        start = min(start, i)
        self.head_start = start
        return start

    def prototype_shape(self, img_size=None) -> Tuple[int, int, int]:
        """(tokens, dim, 1) of the token map at the cut (always computed on the internal 224x224 resize)."""
        if self.head_start == 0:
            return 3, 224, 224
        g = self.base.patch_grid[0] // (2 ** self.head_start)
        return g * g, int(self.base.embed_dim * 2 ** self.head_start), 1

    def _resize(self, x: torch.Tensor) -> torch.Tensor:
        if x.shape[-2:] != (224, 224):
            x = F.interpolate(x, size=(224, 224), mode="bilinear", align_corners=False, antialias=True)
        return x

    def forward_trunk(self, x: torch.Tensor) -> torch.Tensor:
        x = self._resize(x)
        if self.head_start == 0:
            return x
        return self.base.run_layers(self.base.embed(x), 0, self.head_start)

    def forward_head(self, tokens: torch.Tensor):
        if self.head_start == 0:
            tokens = self.base.embed(tokens)
        global_feat = self.base.pool(self.base.run_layers(tokens, self.head_start, self.base.num_layers))
        feat = self.bottleneck(global_feat) if self.neck == "bnneck" else global_feat
        if self.training:
            return self.classifier(feat), global_feat
        return global_feat

    def forward(self, x: torch.Tensor):
        return self.forward_head(self.forward_trunk(x))


def _make(name: str):
    def ctor(**kwargs):
        return SwinTransformerReID(model_name=name, **kwargs)
    return ctor


swin_transformer_tiny = _make("swin_tiny")
swin_transformer_small = _make("swin_small")
swin_transformer_base = _make("swin_base")
swin_transformer_large = _make("swin_large")

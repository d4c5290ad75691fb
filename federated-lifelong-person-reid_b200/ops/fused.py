"""Fused memory-bound ops of the local step (``csrc/fused_ops.cu``): flat-arena optimizers with the
continual-learning penalty folded in, importance accumulation, label-smoothing CE, NHWC batch-norm, pooling."""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.nn.functional as F

from . import native

# (tests: ``native.use_emulated_libraries`` sends CPU tensors down the kernel paths below - tests/emu)
use_emulated_libraries = native.use_emulated_libraries
_emu_libs = native._emu_libs
_lib = native.kernels
_native = native.on_device
_stream = native.stream_of


# --------------------------------------------------------------------------------------------- optimizers
def _opt_stats_scratch(device) -> torch.Tensor:
    """Per-block partials of the optimizer's penalty statistics (2 per block, at most 132 * 8 blocks), summed by the
    library in block order so that the reported penalty is reproducible."""
    return torch.empty(2 * 132 * 8, dtype=torch.float32, device=device)


def fused_optimizer_step(kind: str, p: torch.Tensor, g: torch.Tensor, m: Optional[torch.Tensor],
                         v: Optional[torch.Tensor], *, lr: float, step: int, beta1: float = 0.9, beta2: float = 0.999,
                         eps: float = 1e-8, weight_decay: float = 0.0, momentum: float = 0.0,
                         Q: Optional[torch.Tensor] = None, R: Optional[torch.Tensor] = None, lam2: float = 0.0,
                         penalty_ones: bool = False, G: Optional[torch.Tensor] = None, lam1: float = 0.0,
                         atten: float = 0.0, p_bf16: Optional[torch.Tensor] = None,
                         stats: Optional[torch.Tensor] = None, hyper: Optional[torch.Tensor] = None,
                         anchor: Optional[torch.Tensor] = None, anchor_m: Optional[torch.Tensor] = None,
                         anchor_v: Optional[torch.Tensor] = None) -> None:
    """One in-place optimizer step over a flat fp32 arena.

    gradient used:  g + wd * (p - atten*G) + 2*lam2*(Q*p - R) + lam1*sign(p - G)
    (``Q``/``R`` encode EWC / MAS / FedProx / FedCurv penalties, ``G`` is FedSTIL's global weight;
    ``stats[0] += sum(Q p^2 - 2 R p)``, ``stats[1] += sum|p - G|`` are the penalty values for loss reporting).

    ``anchor`` (CUDA only; the CPU twin is ``ArenaOptimizer._anchor_step``): FedSTIL's *trained* L1 anchor
    ``theta0 = atten*G + aw0`` replaces ``G`` in the L1 term and is itself stepped in the same pass with gradient
    ``-lam1*sign(p - theta0) + wd*(theta0 - atten*G)`` and its own moments (reference ``fedstil.py:53-76,639-647``).
    """
    adam = kind == "adam"
    if hyper is not None and not _native(p):
        lr, step = float(hyper[0]), int(hyper[1])
    if not _native(p):
        assert anchor is None, "the CPU path of the trained anchor is ArenaOptimizer._anchor_step"
        with torch.no_grad():
            grad = g.clone()
            base = p
            if G is not None:
                d = p - G
                if stats is not None:
                    stats[1] += d.abs().sum()
                grad += lam1 * torch.sign(d)
                base = p - atten * G
            if R is not None:
                q = torch.ones_like(p) if penalty_ones or Q is None else Q
                if stats is not None:
                    stats[0] += (q * p * p - 2 * R * p).sum()
                grad += 2 * lam2 * (q * p - R)
            grad += weight_decay * base
            if adam:
                m.mul_(beta1).add_(grad, alpha=1 - beta1)
                v.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
                bc1 = 1 - beta1 ** step
                bc2 = 1 - beta2 ** step
                denom = v.sqrt() / math.sqrt(bc2) + eps
                p.addcdiv_(m, denom, value=-lr / bc1)
            else:
                if momentum != 0.0:
                    m.mul_(momentum).add_(grad)
                    grad = m
                p.add_(grad, alpha=-lr)
            if p_bf16 is not None:
                p_bf16.copy_(p)
        return
    lib = _lib()
    rc = lib.flpr_fused_opt(int(adam), native.ptr(p), native.ptr(g), native.ptr(m), native.ptr(v), native.ptr(Q),
                            native.ptr(R), native.ptr(G), native.ptr(p_bf16), native.ptr(stats), p.numel(), lr, beta1,
                            beta2, eps, weight_decay, int(step), lam2, lam1, atten, momentum, int(penalty_ones),
                            native.ptr(hyper), native.ptr(anchor if G is not None else None), native.ptr(anchor_m),
                            native.ptr(anchor_v), native.ptr(None if stats is None else _opt_stats_scratch(p.device)),
                            _stream(p.device))
    native.check(rc, "flpr_fused_opt")
    native.count_launch()


def importance_accumulate(Fbuf: torch.Tensor, g: torch.Tensor, scale: float, mode: str = "fisher") -> None:
    """``F += scale * g**2`` (fisher) or ``F += scale * |g|`` (mas)."""
    if not _native(Fbuf):
        with torch.no_grad():
            Fbuf.add_((g * g) if mode == "fisher" else g.abs(), alpha=scale)
        return
    lib = _lib()
    rc = lib.flpr_importance_accum(native.ptr(Fbuf), native.ptr(g), Fbuf.numel(), scale, 0 if mode == "fisher" else 1,
                                   _stream(Fbuf.device))
    native.check(rc, "flpr_importance_accum")
    native.count_launch()


def cast_bf16(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    if out is None:
        out = torch.empty_like(x, dtype=torch.bfloat16)
    if not _native(x) or x.numel() % 4 or not x.is_contiguous():
        out.copy_(x)
        return out
    lib = _lib()
    native.check(lib.flpr_cast_bf16(native.ptr(x), native.ptr(out), x.numel(), _stream(x.device)), "flpr_cast_bf16")
    native.count_launch()
    return out


def compose_adaptive(G: torch.Tensor, A: torch.Tensor, atten: float, theta: Optional[torch.Tensor] = None,
                     theta_bf16: Optional[torch.Tensor] = None) -> None:
    """theta = atten * G + A (FedSTIL adaptive compose, ``methods/fedstil.py:85``) with optional bf16 copy."""
    if not _native(G):
        t = atten * G + A
        if theta is not None:
            theta.copy_(t)
        if theta_bf16 is not None:
            theta_bf16.copy_(t)
        return
    lib = _lib()
    native.check(lib.flpr_compose(native.ptr(G), native.ptr(A), atten, native.ptr(theta), native.ptr(theta_bf16),
                                  G.numel(), _stream(G.device)), "flpr_compose")
    native.count_launch()


# --------------------------------------------------------------------------------------------- losses
def ce_label_smooth_reference(logits: torch.Tensor, target: torch.Tensor, eps: float) -> torch.Tensor:
    """fp32 reference of ``criterions/cross_entropy.py:35-40``."""
    logp = F.log_softmax(logits.float(), dim=1)
    c = logits.shape[1]
    t = torch.zeros_like(logp).scatter_(1, target.view(-1, 1), 1.0)
    t = (1 - eps) * t + eps / c
    return (-t * logp).mean(0).sum()


class _CELabelSmoothFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, target, eps, stats):
        b, c = logits.shape
        dlogits = torch.empty_like(logits)
        local = torch.zeros(2 + 2 * b, dtype=torch.float32, device=logits.device)   # [loss, hits] + per-row scratch
        lib = _lib()
        rc = lib.flpr_ce_label_smooth(native.ptr(logits), native.ptr(target), native.ptr(dlogits), native.ptr(local),
                                      native.ptr(local[2:]), b,
                                      c, logits.stride(0), eps, 1.0 / b, int(logits.dtype == torch.bfloat16),
                                      int(dlogits.dtype == torch.bfloat16), _stream(logits.device))
        native.check(rc, "flpr_ce_label_smooth")
        native.count_launch()
        if stats is not None:
            stats += local[:2]
        ctx.save_for_backward(dlogits)
        return local[0]

    @staticmethod
    def backward(ctx, gout):
        (dlogits,) = ctx.saved_tensors
        return dlogits * gout.to(dlogits.dtype), None, None, None


def ce_label_smooth(logits: torch.Tensor, target: torch.Tensor, eps: float = 0.1,
                    stats: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Label-smoothing cross entropy. ``stats`` (float[2], optional) accumulates [loss, #top-1 hits] on device, which
    replaces the per-step ``.cpu().item()`` syncs of ``methods/baseline.py:47-48``."""
    if not _native(logits):
        loss = ce_label_smooth_reference(logits, target, eps)
        if stats is not None:
            with torch.no_grad():
                stats[0] += loss.detach()
                stats[1] += (logits.argmax(1) == target).sum()
        return loss
    assert logits.stride(1) == 1 and logits.dtype in (torch.bfloat16, torch.float32)
    return _CELabelSmoothFn.apply(logits, target.long().contiguous(), float(eps), stats)


# --------------------------------------------------------------------------------------------- batch norm (NHWC)
class _BNTrainFn(torch.autograd.Function):
    """Training-mode batch norm over ``[M, C]`` bf16 (NHWC flattened), optional fused residual add + ReLU."""

    @staticmethod
    def forward(ctx, x, gamma, beta, running_mean, running_var, residual, eps, momentum, relu, pre_part=None,
                ggrad=None, bgrad=None):
        """``ggrad`` / ``bgrad``: the affine parameters' slots in the zeroed flat gradient arena; when given, the
        backward kernel accumulates dgamma / dbeta straight into them (no temporaries, no AccumulateGrad adds)."""
        m, c = x.shape
        dev = x.device
        y = torch.empty_like(x)
        lib = _lib()
        scratch = torch.empty(6, c, dtype=torch.float32, device=dev)  # -, -, mean, rstd, scale, shift
        if pre_part is None:
            part = torch.empty(lib.flpr_bn_partials_floats(m, c), dtype=torch.float32, device=dev)
            npre = 0
        else:                       # statistics already reduced to column partials by the convolution's epilogue
            part, npre = None, pre_part.shape[0]
            assert pre_part.is_contiguous() and pre_part.shape[1:] == (2, c)
        rc = lib.flpr_bn_fwd(native.ptr(x), native.ptr(gamma), native.ptr(beta), native.ptr(residual), native.ptr(y),
                             native.ptr(part), native.ptr(scratch[2]),
                             native.ptr(scratch[3]), native.ptr(scratch[4]), native.ptr(scratch[5]),
                             native.ptr(running_mean), native.ptr(running_var), m, c, eps, momentum, int(relu),
                             native.ptr(pre_part), npre, _stream(dev))
        native.check(rc, "flpr_bn_fwd")
        native.count_launch(3 if pre_part is None else 2)
        ctx.save_for_backward(x, y, gamma, scratch)
        ctx.relu = relu
        ctx.has_res = residual is not None
        ctx.slots = (ggrad, bgrad)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, y, gamma, scratch = ctx.saved_tensors
        m, c = x.shape
        dy = dy.contiguous()
        ggrad, bgrad = ctx.slots
        direct = ggrad is not None
        dgb = None if direct else torch.empty(2, c, dtype=torch.float32, device=x.device)
        dx = torch.empty_like(x)
        dres = torch.empty_like(x) if ctx.has_res else None
        lib = _lib()
        part = torch.empty(lib.flpr_bn_partials_floats(m, c), dtype=torch.float32, device=x.device)
        rc = lib.flpr_bn_bwd(native.ptr(dy), native.ptr(y), native.ptr(x), native.ptr(scratch[2]),
                             native.ptr(scratch[3]), native.ptr(gamma),
                             native.ptr(ggrad if direct else dgb[0]), native.ptr(bgrad if direct else dgb[1]),
                             native.ptr(part), native.ptr(dres), native.ptr(dx), m, c, int(ctx.relu), int(direct),
                             _stream(x.device))
        native.check(rc, "flpr_bn_bwd")
        native.count_launch(3)
        if direct:
            return dx, None, None, None, None, dres, None, None, None, None, None, None
        return dx, dgb[0], dgb[1], None, None, dres, None, None, None, None, None, None


def batch_norm_nhwc(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, running_mean: Optional[torch.Tensor],
                    running_var: Optional[torch.Tensor], *, training: bool, eps: float = 1e-5, momentum: float = 0.1,
                    relu: bool = False, residual: Optional[torch.Tensor] = None,
                    pre_part: Optional[torch.Tensor] = None, grad_slots=None) -> torch.Tensor:
    """BatchNorm over ``[M, C]`` (channels last) with fused residual + ReLU. fp32 affine parameters.
    ``pre_part`` ``[P, 2, C]``: column partials (sum, sum of squares) of the producer's fp32 output, written by the
    GEMM / conv epilogue; when given, the statistics pass over ``x`` is skipped."""
    if not _native(x):
        xf = x.float()
        if training:
            if pre_part is not None:
                n = xf.shape[0]
                mean = pre_part[:, 0].sum(0) / n
                var = (pre_part[:, 1].sum(0) / n - mean * mean).clamp_min(0)
            else:
                mean = xf.mean(0)
                var = xf.var(0, unbiased=False)
            if running_mean is not None:
                with torch.no_grad():
                    n = xf.shape[0]
                    running_mean.mul_(1 - momentum).add_(mean.detach(), alpha=momentum)
                    running_var.mul_(1 - momentum).add_(var.detach() * (n / max(n - 1, 1)), alpha=momentum)
        else:
            mean, var = running_mean, running_var
        y = (xf - mean) * torch.rsqrt(var + eps) * gamma + beta
        if residual is not None:
            y = y + residual.float()
        if relu:
            y = torch.relu(y)
        return y.to(x.dtype)
    x = x.contiguous()
    if training:
        gg, bg = grad_slots if grad_slots is not None else (None, None)
        if gg is None or bg is None or not gamma.requires_grad or not beta.requires_grad:
            gg = bg = None                        # both or neither (e.g. the BNNeck bias is frozen)
        return _BNTrainFn.apply(x, gamma, beta, running_mean, running_var, residual, eps, momentum, relu, pre_part,
                                gg, bg)
    scale = gamma * torch.rsqrt(running_var + eps)
    shift = beta - running_mean * scale
    return affine_act(x, scale, shift, relu=relu, residual=residual)


def affine_act(x: torch.Tensor, scale: torch.Tensor, shift: torch.Tensor, *, relu: bool = False,
               residual: Optional[torch.Tensor] = None) -> torch.Tensor:
    """y = relu?(x * scale[c] + shift[c] (+ residual)) over ``[M, C]`` bf16 (inference-mode BN)."""
    if not _native(x):
        y = x.float() * scale + shift
        if residual is not None:
            y = y + residual.float()
        return (torch.relu(y) if relu else y).to(x.dtype)
    m, c = x.shape
    y = torch.empty_like(x)
    lib = _lib()
    scale_f, shift_f = scale.float().contiguous(), shift.float().contiguous()          # (kept alive over the call)
    rc = lib.flpr_affine_act(native.ptr(x), native.ptr(scale_f),
                             native.ptr(shift_f), native.ptr(residual), native.ptr(y), m, c,
                             int(relu), _stream(x.device))
    native.check(rc, "flpr_affine_act")
    native.count_launch()
    return y


class _GapFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        n, hw, c = x.shape
        out = torch.empty(n, c, dtype=torch.float32, device=x.device)
        lib = _lib()
        native.check(lib.flpr_gap_fwd(native.ptr(x), native.ptr(out), None, n, hw, c, _stream(x.device)),
                     "flpr_gap_fwd")
        native.count_launch()
        ctx.shape = (n, hw, c)
        return out

    @staticmethod
    def backward(ctx, dout):
        n, hw, c = ctx.shape
        dx = torch.empty(n, hw, c, dtype=torch.bfloat16, device=dout.device)
        lib = _lib()
        dout_f = dout.float().contiguous()
        native.check(lib.flpr_gap_bwd(native.ptr(dout_f), native.ptr(dx), n, hw, c,
                                      _stream(dout.device)), "flpr_gap_bwd")
        native.count_launch()
        return dx


def global_avg_pool_nhwc(x: torch.Tensor) -> torch.Tensor:
    """``[N, HW, C]`` bf16 -> ``[N, C]`` fp32."""
    if not _native(x):
        return x.float().mean(1)
    return _GapFn.apply(x.contiguous())


# --------------------------------------------------------------------------------------------- Swin window attention
class _WindowAttnFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, bias, scale):
        bw, n, three, h, d = qkv.shape
        lib = _lib()
        qkv = qkv.contiguous()
        bias = bias.float().contiguous()
        out = torch.empty(bw, n, h * d, dtype=qkv.dtype, device=qkv.device)
        rc = lib.flpr_window_attn_fwd(native.ptr(qkv), native.ptr(bias), native.ptr(out), bw, n, h, d, bias.shape[0],
                                      float(scale), int(qkv.dtype == torch.bfloat16), _stream(qkv.device))
        native.check(rc, "flpr_window_attn_fwd")
        native.count_launch()
        ctx.save_for_backward(qkv, bias)
        ctx.scale = float(scale)
        return out

    @staticmethod
    def backward(ctx, dout):
        qkv, bias = ctx.saved_tensors
        bw, n, three, h, d = qkv.shape
        lib = _lib()
        dout = dout.contiguous().to(qkv.dtype)
        dqkv = torch.empty_like(qkv)
        dbias = torch.zeros_like(bias) if ctx.needs_input_grad[1] else None
        rc = lib.flpr_window_attn_bwd(native.ptr(qkv), native.ptr(bias), native.ptr(dout), native.ptr(dqkv),
                                      native.ptr(dbias), bw, n, h, d, bias.shape[0], ctx.scale,
                                      int(qkv.dtype == torch.bfloat16), _stream(qkv.device))
        native.check(rc, "flpr_window_attn_bwd")
        native.count_launch()
        return dqkv, dbias, None


def window_attention_supported(qkv: torch.Tensor) -> bool:
    return _native(qkv) and qkv.dim() == 5 and qkv.shape[1] <= 64 and qkv.shape[4] <= 64 and \
        qkv.dtype in (torch.bfloat16, torch.float32)


def window_attention(qkv: torch.Tensor, bias: torch.Tensor, scale: float) -> torch.Tensor:
    """Fused window attention (``models/swin_transformer.py:255-286``). ``qkv``: ``[BW, N, 3, heads, D]``, ``bias``:
    ``[nW or 1, heads, N, N]`` (relative-position bias + shift mask; window index = ``bw % nW``). Returns
    ``[BW, N, heads*D]``. CPU / unsupported shapes: plain tensor ops."""
    if window_attention_supported(qkv):
        return _WindowAttnFn.apply(qkv, bias, scale)
    bw, n, _, h, d = qkv.shape
    q, k, v = qkv.float().permute(2, 0, 3, 1, 4)                   # [BW, H, N, D]
    nwb = bias.shape[0]
    s = (q * scale) @ k.transpose(-1, -2)
    s = s.view(bw // nwb, nwb, h, n, n) + bias.float().unsqueeze(0)
    p = torch.softmax(s.view(bw, h, n, n), dim=-1)
    return (p @ v).transpose(1, 2).reshape(bw, n, h * d).to(qkv.dtype)


# --------------------------------------------------------------------------------------------- metric / KD losses
class _MinedDistancesFn(torch.autograd.Function):
    """``(dist_ap, dist_an)`` of the fast-reid triplet loss (``criterions/triplet_loss.py:89-127``): Gram matrix on the
    wgmma GEMM (bf16 hi / lo split: ~fp32 accuracy, the distances are differences of large numbers), distance row +
    masks + hard / softmax-weighted mining in one kernel per anchor; backward = one small kernel that folds the mining
    Jacobians with the incoming gradients into ``S = W + W^T`` and ONE wgmma GEMM ``S @ X``."""

    @staticmethod
    def forward(ctx, x, labels, cosine, hard):
        from .rank import similarity
        lib = _lib()
        xf = x.float().contiguous()
        b = xf.shape[0]
        dev = xf.device
        G = similarity(xf, xf, precise=True)                                  # [B, B] fp32
        sq = (xf * xf).sum(1) if not cosine else None
        dist_ap = torch.empty(b, dtype=torch.float32, device=dev)
        dist_an = torch.empty(b, dtype=torch.float32, device=dev)
        jap = torch.empty(b, b, dtype=torch.float32, device=dev)
        jan = torch.empty(b, b, dtype=torch.float32, device=dev)
        lab = labels.to(dev).long().contiguous()
        rc = lib.flpr_triplet_mine_fwd(native.ptr(G), G.stride(0), native.ptr(sq), native.ptr(lab), b, int(cosine),
                                       int(hard), native.ptr(dist_ap), native.ptr(dist_an), native.ptr(jap),
                                       native.ptr(jan), _stream(dev))
        native.check(rc, "flpr_triplet_mine_fwd")
        native.count_launch()
        ctx.save_for_backward(xf, jap, jan)
        ctx.cosine = bool(cosine)
        ctx.in_dtype = x.dtype
        return dist_ap, dist_an

    @staticmethod
    def backward(ctx, g_ap, g_an):
        from .gemm import gemm
        xf, jap, jan = ctx.saved_tensors
        b, d = xf.shape
        dev = xf.device
        lib = _lib()
        lds = (b + 7) // 8 * 8
        S = torch.empty(b, lds, dtype=torch.bfloat16, device=dev)
        rs = torch.empty(b, dtype=torch.float32, device=dev)
        g_ap = (g_ap if g_ap is not None else torch.zeros(b, device=dev)).float().contiguous()
        g_an = (g_an if g_an is not None else torch.zeros(b, device=dev)).float().contiguous()
        rc = lib.flpr_triplet_mine_bwd(native.ptr(jap), native.ptr(jan), native.ptr(g_ap), native.ptr(g_an), b,
                                       native.ptr(S), lds, native.ptr(rs), _stream(dev))
        native.check(rc, "flpr_triplet_mine_bwd")
        native.count_launch()
        xb = xf.to(torch.bfloat16)
        if lds != b:
            xb = torch.nn.functional.pad(xb, (0, 0, 0, lds - b))
        # S [B, K = B'] (K-major) x X [K = B', N = D] (MN-major): fp32 out; hi / lo split of X keeps fp32-level accuracy
        sx = gemm(S, xb, b_kmajor=False, out_dtype=torch.float32)
        x_lo = (xf - xf.to(torch.bfloat16).float()).to(torch.bfloat16)
        if lds != b:
            x_lo = torch.nn.functional.pad(x_lo, (0, 0, 0, lds - b))
        sx = sx + gemm(S, x_lo, b_kmajor=False, out_dtype=torch.float32)
        if ctx.cosine:
            dx = -sx                                                           # d(1 - <xi, xj>) / d xi = -xj
        else:
            dx = 2.0 * (rs[:, None] * xf - sx)                                 # d|xi - xj|^2 / d xi = 2 (xi - xj)
        return dx.to(ctx.in_dtype), None, None, None


def mined_distances(x: torch.Tensor, labels: torch.Tensor, cosine: bool, hard: bool):
    """``(dist_ap, dist_an)`` for a feature batch ``x`` ``[B, D]`` (already L2-normalised when ``cosine``)."""
    return _MinedDistancesFn.apply(x, labels, cosine, hard)


def mined_distances_supported(x: torch.Tensor) -> bool:
    return _native(x) and x.dim() == 2 and x.shape[1] % 8 == 0 and 2 <= x.shape[0] <= 4096


class _KDKLFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, s, t, temperature):
        lib = _lib()
        s, t = s.contiguous(), t.contiguous().to(s.dtype)
        b, c = s.shape
        ds = torch.empty(b, c, dtype=torch.float32, device=s.device)
        loss = torch.zeros(1, dtype=torch.float32, device=s.device)
        rc = lib.flpr_kd_kl(native.ptr(s), native.ptr(t), native.ptr(ds), native.ptr(loss), b, c, s.stride(0),
                            t.stride(0), float(temperature), int(s.dtype == torch.bfloat16), _stream(s.device))
        native.check(rc, "flpr_kd_kl")
        native.count_launch()
        ctx.save_for_backward(ds)
        ctx.in_dtype = s.dtype
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        (ds,) = ctx.saved_tensors
        return (ds * g).to(ctx.in_dtype), None, None


def kd_kl(student: torch.Tensor, teacher: torch.Tensor, temperature: float) -> torch.Tensor:
    """``KL(softmax(t/T) || softmax(s/T)) * T^2 / B`` (``criterions/kd_loss.py:10-27``), fused forward + gradient."""
    if not _native(student) or student.dtype not in (torch.float32, torch.bfloat16):
        T = temperature
        p_s = F.log_softmax(student.float() / T, dim=1)
        p_t = F.softmax(teacher.float() / T, dim=1)
        return F.kl_div(p_s, p_t, reduction="sum") * (T ** 2) / student.shape[0]
    return _KDKLFn.apply(student, teacher.detach(), temperature)


class _BCEDistillFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z, target, prev):
        lib = _lib()
        z = z.contiguous()
        b, c = z.shape
        p = 0 if prev is None else min(int(prev.shape[1]), c)
        prev_f = None if prev is None else prev.float().contiguous()
        dz = torch.empty(b, c, dtype=torch.float32, device=z.device)
        loss = torch.zeros(1, dtype=torch.float32, device=z.device)
        target_l = target.to(z.device).long().contiguous()
        rc = lib.flpr_bce_distill(native.ptr(z), native.ptr(target_l),
                                  native.ptr(prev_f), native.ptr(dz), native.ptr(loss), b, c, p, z.stride(0),
                                  0 if prev_f is None else prev_f.stride(0), int(z.dtype == torch.bfloat16),
                                  _stream(z.device))
        native.check(rc, "flpr_bce_distill")
        native.count_launch()
        ctx.save_for_backward(dz)
        ctx.in_dtype = z.dtype
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        (dz,) = ctx.saved_tensors
        return (dz * g).to(ctx.in_dtype), None, None


def bce_distill(score: torch.Tensor, target: torch.Tensor, prev_logits: Optional[torch.Tensor]) -> torch.Tensor:
    """iCaRL's distillation-pass loss (``methods/icarl.py:226-234``): ``BCEWithLogits(score, onehot(target))`` +
    ``BCEWithLogits(score[:, :P], sigmoid(prev_logits))`` (both mean-reduced), one fused kernel with gradient."""
    if not _native(score) or score.dtype not in (torch.float32, torch.bfloat16):
        z = score.float()
        onehot = torch.zeros_like(z).scatter_(1, target.view(-1, 1).to(z.device), 1.0)
        loss = F.binary_cross_entropy_with_logits(z, onehot)
        if prev_logits is not None:
            p = min(prev_logits.shape[1], z.shape[1])
            loss = loss + F.binary_cross_entropy_with_logits(z[:, :p], torch.sigmoid(prev_logits[:, :p].float()))
        return loss
    return _BCEDistillFn.apply(score, target, None if prev_logits is None else prev_logits.detach())

"""Tensor-core GEMM / implicit-GEMM convolution ops (``csrc/gemm_wgmma.cu``) and their autograd wrappers.

Layout conventions: activations are NHWC bf16 flattened to ``[pixels, channels]``; weights are ``[out, in]`` (1x1 /
linear) or ``[out, kh, kw, in]`` (3x3, "OHWI"), i.e. the reduction dim is always contiguous in the forward pass. The
backward passes reuse the same kernel in its MN-major operand modes, so no tensor is ever transposed in memory.

Reference call sites replaced: ``models/resnet.py:121-141`` (bottleneck convs), ``models/resnet.py:321``
(classifier), ``tools/evaluate.py:100`` (gallery x query similarity).
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from . import native


def _bf(x: torch.Tensor) -> torch.Tensor:
    return x if x.dtype == torch.bfloat16 else x.to(torch.bfloat16)


def col_part_rows(m: int) -> int:
    """Number of partial rows the GEMM epilogue writes for ``m`` output rows (4 epilogue warps per 128-row tile)."""
    return ((m + 127) // 128) * 4


def col_part_buffer(m: int, n: int, device) -> torch.Tensor:
    return torch.empty(col_part_rows(m), 2, n, dtype=torch.float32, device=device)


def _split_workspace(split: int, rows: int, ld: int, device) -> Optional[torch.Tensor]:
    """Partial-product slices of a split-K GEMM (reduced in split order by the library: bitwise reproducible)."""
    if split <= 1:
        return None
    return torch.empty(split * ((rows * ld + 3) // 4 * 4), dtype=torch.float32, device=device)


def _check_epilogue(split_k: int, col_part, bias, bias_m, residual, relu: bool) -> None:
    """Option combinations the kernel cannot compute as one result; refused alike on both devices. A split-K GEMM
    would run the epilogue once per split (bias added ``split_k`` times, ReLU of each partial), and ``col_part`` holds
    the statistics of the stored ``alpha * A@B^T``, which has no bias / residual / ReLU."""
    epi = bias is not None or bias_m is not None or residual is not None or relu
    if split_k > 1 and epi:
        raise ValueError("split_k > 1 takes no bias / residual / ReLU epilogue")
    if col_part is not None and epi:
        raise ValueError("col_part takes no bias / residual / ReLU epilogue")


def _col_part_reference(d: torch.Tensor, col_part: torch.Tensor) -> None:
    """CPU reference of the fused statistics: 32-row partial sums of ``d`` and ``d*d`` (``d`` as stored, i.e.
    already rounded to the output dtype)."""
    m, n = d.shape
    rows = col_part.shape[0]
    pad = rows * 32 - m
    dd = torch.cat([d.float(), d.new_zeros(pad, n).float()]) if pad else d.float()
    dd = dd.view(rows, 32, n)
    col_part[:, 0].copy_(dd.sum(1))
    col_part[:, 1].copy_((dd * dd).sum(1))


def gemm(a: torch.Tensor, b: torch.Tensor, *, a_kmajor: bool = True, b_kmajor: bool = True,
         out_dtype: torch.dtype = torch.bfloat16, trans_out: bool = False, alpha: float = 1.0,
         bias_n: Optional[torch.Tensor] = None, bias_m: Optional[torch.Tensor] = None, relu: bool = False,
         residual: Optional[torch.Tensor] = None, split_k: int = 1, bn: int = 0,
         out: Optional[torch.Tensor] = None, col_part: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``D[M,N] = alpha * A @ B^T`` with bf16 operands and fp32 accumulation.

    ``a`` is ``[M,K]`` (``a_kmajor``) or ``[K,M]``; ``b`` is ``[N,K]`` (``b_kmajor``) or ``[K,N]``.
    Returns ``[M,N]`` (``[N,M]`` when ``trans_out``). ``out`` (optional) is overwritten, whatever ``split_k``.
    ``split_k > 1`` needs an fp32 output and no bias / residual / ReLU (the splits are summed in a fixed order, so the
    result is reproducible).
    ``col_part`` (fp32 ``[ceil(M/128)*4, 2, N]``, see :func:`col_part_buffer`) receives per-32-row partial column
    sums / sums of squares of the stored ``alpha * A@B^T`` (rows past ``M`` count as 0): the batch-norm statistics
    pass over the output is fused away. It takes no bias / residual / ReLU.
    """
    M, K = (a.shape if a_kmajor else (a.shape[1], a.shape[0]))
    N, Kb = (b.shape if b_kmajor else (b.shape[1], b.shape[0]))
    assert K == Kb, f"reduction dims differ: {K} vs {Kb}"
    _check_epilogue(split_k, col_part, bias_n, bias_m, residual, relu)
    if not a.is_cuda:
        A = a.float() if a_kmajor else a.float().t()
        B = b.float() if b_kmajor else b.float().t()
        A, B = A.to(torch.bfloat16).float(), B.to(torch.bfloat16).float()
        d = alpha * (A @ B.t())
        if col_part is not None:
            _col_part_reference(d.to(out_dtype), col_part)
        if bias_n is not None:
            d = d + bias_n.float()[None, :]
        if bias_m is not None:
            d = d + bias_m.float()[:, None]
        if trans_out:
            d = d.t()
        if residual is not None:
            d = d + residual.float()
        if relu:
            d = torch.relu(d)
        d = d.to(out_dtype).contiguous()
        if out is not None:
            out.copy_(d)
            return out
        return d

    lib = native.load()
    a, b = _bf(a), _bf(b)
    assert a.stride(-1) == 1 and b.stride(-1) == 1, "operands must be row-major"
    lda, ldb = a.stride(0), b.stride(0)
    oshape = (N, M) if trans_out else (M, N)
    if out is None:
        out = torch.empty(oshape, dtype=torch.float32 if split_k > 1 else out_dtype, device=a.device)
    assert out.stride(-1) == 1
    if split_k > 1:
        assert out.dtype == torch.float32
    if residual is not None:
        assert residual.dtype == torch.bfloat16 and residual.shape == out.shape and residual.stride() == out.stride()
    rc = lib.flpr_gemm_bf16(native.ptr(a), native.ptr(b), native.ptr(out), M, N, K, lda, ldb, out.stride(0),
                            0 if a_kmajor else 1, 0 if b_kmajor else 1, int(out.dtype == torch.bfloat16),
                            int(trans_out), float(alpha), native.ptr(bias_n), native.ptr(bias_m), int(relu),
                            native.ptr(residual), int(split_k), int(bn), native.ptr(col_part),
                            native.ptr(_split_workspace(split_k, oshape[0], out.stride(0), a.device)),
                            native.stream(a.device))
    native.check(rc, "flpr_gemm_bf16")
    native.count_launch()
    return out


def conv_nhwc(x: torch.Tensor, w: torch.Tensor, *, padding: int = 1, out_dtype: torch.dtype = torch.bfloat16,
              alpha: float = 1.0, bias: Optional[torch.Tensor] = None, relu: bool = False,
              residual: Optional[torch.Tensor] = None, bn: int = 0,
              col_part: Optional[torch.Tensor] = None, stride: int = 1) -> torch.Tensor:
    """Convolution (stride 1 or 2) as an implicit GEMM. ``x``: ``[N,H,W,C]`` bf16, ``w``: ``[Cout,KH,KW,C]``.

    Returns ``[N,Ho,Wo,Cout]``. Zero padding is produced by TMA out-of-bounds fill; a stride-2 convolution walks
    the input with TMA element strides (same kernel, same pipeline). ``col_part``: see :func:`gemm` (no bias /
    residual / ReLU with it).
    """
    n, h, wd, c = x.shape
    cout, kh, kw, c2 = w.shape
    assert c == c2
    ho, wo = (h + 2 * padding - kh) // stride + 1, (wd + 2 * padding - kw) // stride + 1
    _check_epilogue(1, col_part, bias, None, residual, relu)
    if not x.is_cuda:
        xx = x.to(torch.bfloat16).float().permute(0, 3, 1, 2)
        ww = w.to(torch.bfloat16).float().permute(0, 3, 1, 2)
        y = alpha * F.conv2d(xx, ww, padding=padding, stride=stride)
        if col_part is not None:
            _col_part_reference(y.permute(0, 2, 3, 1).reshape(-1, cout).to(out_dtype), col_part)
        if bias is not None:
            y = y + bias.float()[None, :, None, None]
        y = y.permute(0, 2, 3, 1)
        if residual is not None:
            y = y + residual.float()
        if relu:
            y = torch.relu(y)
        return y.to(out_dtype).contiguous()
    lib = native.load()
    x, w = _bf(x).contiguous(), _bf(w).contiguous()
    out = torch.empty((n, ho, wo, cout), dtype=out_dtype, device=x.device)
    if residual is not None:
        assert residual.dtype == torch.bfloat16 and residual.is_contiguous() and residual.shape == out.shape
    rc = lib.flpr_conv_nhwc_bf16(native.ptr(x), native.ptr(w), native.ptr(out), n, h, wd, c, cout, kh, kw, padding,
                                 padding, int(out_dtype == torch.bfloat16), float(alpha), native.ptr(bias), int(relu),
                                 native.ptr(residual), int(bn), native.ptr(col_part), int(stride), 0, 0, 0,
                                 native.stream(x.device))
    native.check(rc, "flpr_conv_nhwc_bf16")
    native.count_launch()
    return out


def conv_supported(h: int, w: int, c: int, k: int, stride: int = 1, padding: Optional[int] = None) -> bool:
    """Shape constraints of the implicit-GEMM kernel (C multiple of 64; output rows tile into 128-pixel M tiles)."""
    padding = k // 2 if padding is None else padding
    ho, wo = (h + 2 * padding - k) // stride + 1, (w + 2 * padding - k) // stride + 1
    if c % 64 or stride not in (1, 2) or wo < 1 or wo > 128 or 128 % wo:
        return False
    if ho * wo <= 128:
        return 128 % (ho * wo) == 0
    return ho % (128 // wo) == 0


def conv_dgrad_nhwc(dy: torch.Tensor, w: torch.Tensor, *, padding: int = 1,
                    out_dtype: torch.dtype = torch.bfloat16, bn: int = 0) -> torch.Tensor:
    """Data gradient of a stride-1 convolution from the FORWARD weight ``w`` ``[Cout,KH,KW,Cin]`` (no flipped /
    transposed weight copy: the kernel walks the taps mirrored and reads ``w`` MN-major). ``dy``: ``[N,H,W,Cout]``."""
    n, h, wd, cout = dy.shape
    cout2, kh, kw, cin = w.shape
    assert cout == cout2
    if not dy.is_cuda:
        dd = dy.to(torch.bfloat16).float().permute(0, 3, 1, 2)
        ww = w.to(torch.bfloat16).float().permute(0, 3, 1, 2)                 # [Cout,Cin,KH,KW]
        dx = torch.nn.grad.conv2d_input((n, cin, h, wd), ww, dd, padding=padding)
        return dx.permute(0, 2, 3, 1).to(out_dtype).contiguous()
    lib = native.load()
    dy, w = _bf(dy).contiguous(), _bf(w).contiguous()
    out = torch.empty((n, h, wd, cin), dtype=out_dtype, device=dy.device)
    rc = lib.flpr_conv_dgrad_nhwc_bf16(native.ptr(dy), native.ptr(w), native.ptr(out), n, h, wd, cin, cout, kh, kw,
                                       padding, padding, int(out_dtype == torch.bfloat16), int(bn),
                                       native.stream(dy.device))
    native.check(rc, "flpr_conv_dgrad_nhwc_bf16")
    native.count_launch()
    return out


def _auto_split(m: int, n: int, k: int, taps: int = 1) -> int:
    """split-K factor for weight-gradient GEMMs (small MxN, very long K): aim for ~1-2 CTAs per SM."""
    tiles = ((m + 127) // 128) * ((n + 127) // 128) * taps
    kb = (k + 63) // 64
    if tiles >= 120 or kb < 8:
        return 1
    return max(1, min(kb // 4, (132 + tiles - 1) // tiles))


class _LinearFn(torch.autograd.Function):
    """y[M,N] = x[M,K] @ w[N,K]^T using the bf16 compute copy; gradients: dx bf16, dw fp32 (for the fp32 master).

    When ``grad_out`` (the parameter's slot in the zeroed arena gradient buffer) is given, the weight gradient is
    written straight into it by the GEMM epilogue and ``None`` is returned to autograd: no temporary, no
    ``AccumulateGrad`` read-modify-write pass."""

    @staticmethod
    def forward(ctx, x, w_master, w_bf16, grad_out, want_stats=False, bias=None):
        ctx.save_for_backward(x, w_bf16)
        ctx.w_needs_grad = w_master.requires_grad
        ctx.grad_out = grad_out
        ctx.want_stats = want_stats
        ctx.has_bias = bias is not None
        ctx.set_materialize_grads(False)        # no zero tensor for the (non-differentiable) statistics output
        if not want_stats:
            return gemm(x, w_bf16, bias_n=bias)  # (+ bias[col] in the GEMM epilogue: no separate broadcast-add pass)
        part = col_part_buffer(x.shape[0], w_bf16.shape[0], x.device)
        y = gemm(x, w_bf16, col_part=part)
        ctx.mark_non_differentiable(part)
        return y, part

    @staticmethod
    def backward(ctx, dy, *_):
        if dy is None:
            return None, None, None, None, None, None
        x, w = ctx.saved_tensors
        dy = _bf(dy).contiguous()
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = gemm(dy, w, b_kmajor=False)                               # [M,N] x [N,K]
        if ctx.w_needs_grad:
            m, n, k = w.shape[0], w.shape[1], dy.shape[0]
            split = _auto_split(m, n, k)
            if ctx.grad_out is not None:
                gemm(dy, x, a_kmajor=False, b_kmajor=False, out_dtype=torch.float32, split_k=split, out=ctx.grad_out)
            else:
                dw = gemm(dy, x, a_kmajor=False, b_kmajor=False, out_dtype=torch.float32, split_k=split)
        if ctx.has_bias and ctx.needs_input_grad[5]:
            db = dy.float().sum(0)
        return dx, dw, None, None, None, db


def linear(x: torch.Tensor, w_master: torch.Tensor, w_bf16: Optional[torch.Tensor] = None,
           grad_out: Optional[torch.Tensor] = None, want_stats: bool = False, bias: Optional[torch.Tensor] = None):
    """Linear / 1x1-conv on flattened NHWC activations. ``w_master`` fp32 ``[out,in]`` receives the gradient
    (directly in ``grad_out`` when given - it is overwritten, not accumulated into). ``want_stats`` additionally
    returns the fused batch-norm column partials of the output (``(y, part)``)."""
    if x.is_cuda and (w_master.shape[0] % 8 or w_master.shape[1] % 8 or x.shape[-1] % 8) and not want_stats:
        # TMA needs 16-byte row strides in every operand mode of forward / dgrad / wgrad; a head that is not a
        # multiple of 8 wide (iCaRL grows its classifier by ``n_classes`` at a time, methods/icarl.py) is a tiny GEMM:
        # plain autograd matmul (the fp32 weight gradient lands in the arena slot through AccumulateGrad)
        return F.linear(_bf(x), w_master.to(torch.bfloat16), None if bias is None else bias.to(torch.bfloat16))
    if w_bf16 is None:
        w_bf16 = w_master.detach().to(torch.bfloat16)
    if grad_out is not None and not x.is_cuda:
        grad_out = None
    if bias is not None and (want_stats or bias.dtype != torch.float32 or not bias.is_contiguous()):
        return _LinearFn.apply(_bf(x), w_master, w_bf16, grad_out, want_stats) + bias.to(torch.bfloat16)
    return _LinearFn.apply(_bf(x), w_master, w_bf16, grad_out, want_stats, bias)


class _Conv3x3Fn(torch.autograd.Function):
    """3x3 / stride 1 / pad 1 NHWC convolution: forward, dgrad and wgrad all on the wgmma implicit-GEMM kernel."""

    @staticmethod
    def forward(ctx, x, w_master, w_bf16, grad_out, want_stats=False):
        ctx.save_for_backward(x, w_bf16)
        ctx.w_needs_grad = w_master.requires_grad
        ctx.grad_out = grad_out
        ctx.set_materialize_grads(False)
        if not want_stats:
            return conv_nhwc(x, w_bf16, padding=1)
        n, h, wd, _ = x.shape
        part = col_part_buffer(n * h * wd, w_bf16.shape[0], x.device)
        y = conv_nhwc(x, w_bf16, padding=1, col_part=part)
        ctx.mark_non_differentiable(part)
        return y, part

    @staticmethod
    def backward(ctx, dy, *_):
        if dy is None:
            return None, None, None, None, None
        x, w = ctx.saved_tensors
        dy = _bf(dy).contiguous()
        dx = dw = None
        if ctx.needs_input_grad[0]:
            # dgrad straight from the forward weight: mirrored taps + MN-major B operand inside the kernel
            dx = conv_dgrad_nhwc(dy, w, padding=1)
        if ctx.w_needs_grad:
            if ctx.grad_out is not None:
                conv3x3_wgrad(x, dy, out=ctx.grad_out)
            else:
                dw = conv3x3_wgrad(x, dy)
        return dx, dw, None, None, None


def conv3x3_wgrad(x: torch.Tensor, dy: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """dW[Cout,3,3,Cin] (fp32) = sum over pixels of dy (x) shifted x. ONE launch: grid.z enumerates the 9 filter
    taps (x split-K); the shifted / zero-padded view of ``x`` is produced by 4-D TMA boxes, nothing is copied.
    ``out`` (optional) is overwritten, whatever split factor the shape gets."""
    n, h, w, cin = x.shape
    cout = dy.shape[-1]
    if not x.is_cuda:
        xx = x.float().permute(0, 3, 1, 2)
        dd = dy.float().permute(0, 3, 1, 2)
        g = torch.nn.grad.conv2d_weight(xx, (cout, cin, 3, 3), dd, padding=1)
        g = g.permute(0, 2, 3, 1).contiguous()
        if out is not None:
            out.copy_(g)
            return out
        return g
    lib = native.load()
    x, dy = _bf(x).contiguous(), _bf(dy).contiguous()
    split = _auto_split(cout, cin, n * h * w, taps=9)
    if out is None:
        out = torch.zeros((cout, 3, 3, cin), dtype=torch.float32, device=x.device)
    assert out.is_contiguous() and out.dtype == torch.float32 and out.numel() == cout * 9 * cin
    rc = lib.flpr_conv_wgrad_nhwc_bf16(native.ptr(x), native.ptr(dy), native.ptr(out), n, h, w, cin, cout, 3, 3, 1, 1,
                                       int(split), 0, native.ptr(_split_workspace(split, cout, 9 * cin, x.device)),
                                       native.stream(x.device))
    native.check(rc, "flpr_conv_wgrad_nhwc_bf16")
    native.count_launch()
    return out


def conv3x3(x: torch.Tensor, w_master: torch.Tensor, w_bf16: Optional[torch.Tensor] = None,
            grad_out: Optional[torch.Tensor] = None, want_stats: bool = False):
    if w_bf16 is None:
        w_bf16 = w_master.detach().to(torch.bfloat16)
    if grad_out is not None and not x.is_cuda:
        grad_out = None
    return _Conv3x3Fn.apply(_bf(x), w_master, w_bf16, grad_out, want_stats)


# ------------------------------------------------------------------------------------------------- stride-2 convs
def zero_stuff2(t: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """``[N,Ho,Wo,C]`` -> ``[N,h,w,C]`` with ``t`` at the even positions and zeros elsewhere (the gradient of taking
    every second row / column of an ``h x w`` map)."""
    n, ho, wo, c = t.shape
    assert 2 * (ho - 1) < h and 2 * (wo - 1) < w, "stride-2 map does not fit its stride-1 parent"
    out = t.new_zeros(n, h, w, c)
    out[:, 0:2 * ho:2, 0:2 * wo:2] = t
    return out


def conv_s2_supported(h: int, w: int, cin: int, cout: int, k: int) -> bool:
    """Shapes for which forward, data gradient and weight gradient of a ``k x k`` / stride-2 / pad ``k//2``
    convolution all run on the wgmma kernels (:class:`_ConvStride2Fn`)."""
    if k == 1:
        return cin % 8 == 0 and cout % 8 == 0 and conv_supported(h, w, cin, 1, 2, 0)
    if k != 3:
        return False
    fwd = conv_supported(h, w, cin, 3, 2)
    dgrad = cout % 64 == 0 and cin % 64 == 0 and conv_supported(h, w, cout, 3, 1)     # over the stride-1 parent map
    wgrad = cout % 8 == 0 and w <= 64 and 64 % w == 0 and ((h * w) % 64 == 0 or 64 % (h * w) == 0)
    return fwd and dgrad and wgrad


class _ConvStride2Fn(torch.autograd.Function):
    """``k x k`` (k = 1 or 3) / stride 2 / pad ``k//2`` NHWC convolution with every pass on the wgmma kernels.

    Forward: the implicit-GEMM kernel walks the input with TMA element strides. Backward: a stride-2 convolution is
    its stride-1 parent sampled at the even output positions (``y[i] = z[2i]``), so ``dL/dz`` is ``dy`` zero-stuffed
    to the parent resolution and the validated stride-1 dgrad / wgrad kernels apply unchanged (3x3; the stuffed
    zeros cost 4x the tensor-core work of one layer per ResNet stage - the only strided 3x3 a ResNet stage has).
    1x1: ``dx`` = zero-stuffed ``dy @ W`` and ``dW = dy^T @ x[:, ::2, ::2]`` - two plain GEMMs at the output
    resolution. Reference site: ``models/resnet.py:182`` (``last_stride: 2``) / any head cut above ``layer4``."""

    @staticmethod
    def forward(ctx, x, w_master, w_bf16, grad_out, want_stats=False):
        ctx.save_for_backward(x, w_bf16)
        ctx.w_needs_grad = w_master.requires_grad
        ctx.grad_out = grad_out
        ctx.set_materialize_grads(False)
        k = w_bf16.shape[1]
        if not want_stats:
            return conv_nhwc(x, w_bf16, padding=k // 2, stride=2)
        n, h, wd, _ = x.shape
        ho, wo = (h + 2 * (k // 2) - k) // 2 + 1, (wd + 2 * (k // 2) - k) // 2 + 1
        part = col_part_buffer(n * ho * wo, w_bf16.shape[0], x.device)
        y = conv_nhwc(x, w_bf16, padding=k // 2, stride=2, col_part=part)
        ctx.mark_non_differentiable(part)
        return y, part

    @staticmethod
    def backward(ctx, dy, *_):
        if dy is None:
            return None, None, None, None, None
        x, w = ctx.saved_tensors
        dy = _bf(dy).contiguous()
        n, h, wd, cin = x.shape
        cout, k = w.shape[0], w.shape[1]
        dx = dw = None
        if k == 3:
            dz = zero_stuff2(dy, h, wd)                           # dL/d(stride-1 parent output)
            if ctx.needs_input_grad[0]:
                dx = conv_dgrad_nhwc(dz, w, padding=1)
            if ctx.w_needs_grad:
                if ctx.grad_out is not None:
                    conv3x3_wgrad(x, dz, out=ctx.grad_out)
                else:
                    dw = conv3x3_wgrad(x, dz)
            return dx, dw, None, None, None
        _, ho, wo, _ = dy.shape
        dy2 = dy.reshape(-1, cout)
        if ctx.needs_input_grad[0]:
            dxs = gemm(dy2, w.reshape(cout, cin), b_kmajor=False)             # [N*Ho*Wo, Cin]
            dx = zero_stuff2(dxs.view(n, ho, wo, cin), h, wd)
        if ctx.w_needs_grad:
            xs = x[:, ::2, ::2].contiguous().reshape(-1, cin)                 # the pixels the 1x1 / 2 conv reads
            split = _auto_split(cout, cin, xs.shape[0])
            if ctx.grad_out is not None:
                gemm(dy2, xs, a_kmajor=False, b_kmajor=False, out_dtype=torch.float32, split_k=split,
                     out=ctx.grad_out.reshape(cout, cin))
            else:
                dw = gemm(dy2, xs, a_kmajor=False, b_kmajor=False, out_dtype=torch.float32,
                          split_k=split).view(cout, 1, 1, cin)
        return dx, dw, None, None, None


def conv_stride2(x: torch.Tensor, w_master: torch.Tensor, w_bf16: Optional[torch.Tensor] = None,
                 grad_out: Optional[torch.Tensor] = None, want_stats: bool = False):
    """``x``: ``[N,H,W,Cin]`` bf16, ``w_master``: ``[Cout,k,k,Cin]`` (k = 1 or 3). See :class:`_ConvStride2Fn`."""
    if w_bf16 is None:
        w_bf16 = w_master.detach().to(torch.bfloat16)
    if grad_out is not None and not x.is_cuda:
        grad_out = None
    return _ConvStride2Fn.apply(_bf(x), w_master, w_bf16, grad_out, want_stats)


# ------------------------------------------------------------------------------------------------- ResNet stem
def stem_weight_s2d(w: torch.Tensor) -> torch.Tensor:
    """7x7 / stride-2 stem weight ``[Cout,3,7,7]`` -> ``[Cout, 4, 64]``: the equivalent 4x4 / stride-1 convolution over
    2x2 space-to-depth cells (16 channels per cell: 4 sub-pixels x 3 colours + 4 zeros), 4 cells = one 64-wide K block
    per kernel row. Tap (a, b) of the cell grid covers pixel offsets ``2a + bh - 3`` (a in -2..1, bh in 0..1)."""
    cout = w.shape[0]
    out = w.new_zeros(cout, 4, 4, 16)
    for a in range(4):                       # cell row offset a-2
        for bh in range(2):
            kh = 2 * (a - 2) + bh + 3
            if not 0 <= kh <= 6:
                continue
            for b in range(4):
                for bw in range(2):
                    kw = 2 * (b - 2) + bw + 3
                    if not 0 <= kw <= 6:
                        continue
                    ch = (bh * 2 + bw) * 3
                    out[:, a, b, ch:ch + 3] = w[:, :, kh, kw]
    return out.reshape(cout, 4, 64)


def s2d_pad(x: torch.Tensor) -> torch.Tensor:
    """``[B,H,W,3]`` bf16 -> ``[B, H/2+3, W/2+3, 16]`` bf16 (space-to-depth cells with zero borders)."""
    b, h, w, c = x.shape
    assert c == 3 and h % 2 == 0 and w % 2 == 0
    if not native.on_device(x, "flpr_s2d_pad"):
        y = x.new_zeros(b, h // 2 + 3, w // 2 + 3, 16)
        cells = x.view(b, h // 2, 2, w // 2, 2, 3).permute(0, 1, 3, 2, 4, 5).reshape(b, h // 2, w // 2, 12)
        y[:, 2:2 + h // 2, 2:2 + w // 2, :12] = cells
        return y
    lib = native.kernels()
    x = _bf(x).contiguous()
    y = torch.empty(b, h // 2 + 3, w // 2 + 3, 16, dtype=torch.bfloat16, device=x.device)
    native.check(lib.flpr_s2d_pad(native.ptr(x), native.ptr(y), b, h, w, native.stream_of(x.device)), "flpr_s2d_pad")
    native.count_launch()
    return y


def stem_supported(h: int, w: int) -> bool:
    if h % 2 or w % 2:
        return False
    ho, wo = h // 2, w // 2
    if wo > 128 or 128 % wo:
        return False
    return (128 % (ho * wo) == 0) if ho * wo <= 128 else (ho % (128 // wo) == 0)


def stem_conv(x: torch.Tensor, w4: torch.Tensor, bias: Optional[torch.Tensor], relu: bool = True,
              col_part: Optional[torch.Tensor] = None) -> torch.Tensor:
    """ResNet stem (7x7 / 2 / pad 3 convolution + folded-BN bias + ReLU) on the implicit-GEMM kernel.
    ``x``: ``[B,H,W,3]`` bf16 NHWC, ``w4``: :func:`stem_weight_s2d` of the (folded) weight. Returns ``[B,H/2,W/2,Cout]``.
    ``col_part``: fused batch-norm statistics of the output (train-mode BN after an un-folded stem); it needs
    ``bias=None`` and ``relu=False``."""
    b, h, w, _ = x.shape
    cout = w4.shape[0]
    _check_epilogue(1, col_part, bias, None, None, relu)
    y2 = s2d_pad(x)                                            # [B, H2, W2, 16]
    h2, w2 = h // 2 + 3, w // 2 + 3
    ho, wo = h // 2, w // 2
    if not x.is_cuda:
        win = y2.float().unfold(2, 4, 1)                       # [B, H2, wo, 16, 4] windows of 4 cells
        win = win.permute(0, 1, 2, 4, 3).reshape(b, h2, wo, 64)
        rows = win.unfold(1, 4, 1)                             # [B, ho, wo, 64, 4]
        a = rows.permute(0, 1, 2, 4, 3).reshape(b * ho * wo, 256)
        out = a @ w4.float().reshape(cout, 256).t()
        if col_part is not None:
            _col_part_reference(out.to(torch.bfloat16).float(), col_part)
        if bias is not None:
            out = out + bias.float()
        if relu:
            out = torch.relu(out)
        return out.to(torch.bfloat16).view(b, ho, wo, cout)
    lib = native.load()
    w4 = _bf(w4).contiguous()
    out = torch.empty(b, ho, wo, cout, dtype=torch.bfloat16, device=x.device)
    # the input seen by the conv kernel: [B, H2, wo, 64] with a 16-element (one cell) W stride -> overlapping windows
    rc = lib.flpr_conv_nhwc_bf16(native.ptr(y2), native.ptr(w4), native.ptr(out), b, h2, wo, 64, cout, 4, 1, 0, 0, 1,
                                 1.0, native.ptr(bias), int(relu), None, 0, native.ptr(col_part), 1, 16, w2 * 16,
                                 h2 * w2 * 16, native.stream(x.device))
    native.check(rc, "flpr_conv_nhwc_bf16 (stem)")
    native.count_launch()
    return out


def maxpool3x3s2(x: torch.Tensor) -> torch.Tensor:
    """3x3 / stride 2 / pad 1 max-pool over NHWC bf16."""
    b, h, w, c = x.shape
    if not native.on_device(x, "flpr_maxpool3x3s2"):
        return F.max_pool2d(x.float().permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1).to(x.dtype).contiguous()
    lib = native.kernels()
    x = _bf(x).contiguous()
    y = torch.empty(b, (h - 1) // 2 + 1, (w - 1) // 2 + 1, c, dtype=torch.bfloat16, device=x.device)
    native.check(lib.flpr_maxpool3x3s2(native.ptr(x), native.ptr(y), b, h, w, c, native.stream_of(x.device)),
                 "flpr_maxpool3x3s2")
    native.count_launch()
    return y

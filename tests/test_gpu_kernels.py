"""Numerics of every sm_90a kernel against a plain fp32 PyTorch reference (runs on a GPU box)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, params=["persistent", "classic", "pair", "generic-epilogue"])
def gemm_kernel_variant(request):
    """Every test runs against the wgmma GEMM kernel: persistent grid (default), one CTA per tile, the CTA-pair kernel
    (2-CTA clusters sharing the B tile through TMA multicast) on the shapes it covers, and the generic epilogue forced
    on the shapes that would take the lean one."""
    from flpr_b200.ops import native
    lib = native.load()
    lib.flpr_gemm_set_persistent(0 if request.param == "classic" else 1)
    lib.flpr_gemm_set_pair(1 if request.param == "pair" else 0)       # "persistent" = single-CTA persistent kernel
    lib.flpr_gemm_set_generic_epilogue(1 if request.param == "generic-epilogue" else 0)
    yield request.param
    lib.flpr_gemm_set_persistent(1)
    lib.flpr_gemm_set_pair(-1)
    lib.flpr_gemm_set_generic_epilogue(-1)


def _ref_gemm(a, b):
    return a.to(torch.bfloat16).float() @ b.to(torch.bfloat16).float().t()


def _close(x, ref, rtol=2e-2, atol=None):
    ref = ref.float()
    x = x.float()
    if atol is None:
        atol = 2e-2 * ref.abs().max().item() + 1e-6
    err = (x - ref).abs().max().item()
    assert torch.allclose(x, ref, rtol=rtol, atol=atol), f"max abs err {err} (ref max {ref.abs().max().item()})"


@pytest.mark.parametrize("m,n,k", [(128, 128, 64), (256, 512, 512), (200, 136, 320), (64, 8000, 2048),
                                   (8192, 512, 1024), (8192, 2048, 512), (77, 24, 72)])
@pytest.mark.parametrize("bn", [0, 64, 128, 256])
def test_gemm_kmajor(m, n, k, bn):
    from flpr_b200.ops.gemm import gemm
    torch.manual_seed(0)
    a = torch.randn(m, k, device="cuda")
    b = torch.randn(n, k, device="cuda")
    ref = _ref_gemm(a, b)
    out = gemm(a.bfloat16(), b.bfloat16(), out_dtype=torch.float32, bn=bn)
    _close(out, ref, rtol=1e-3, atol=1e-3 * math.sqrt(k))
    outb = gemm(a.bfloat16(), b.bfloat16(), bn=bn)
    _close(outb, ref)


@pytest.mark.parametrize("amaj,bmaj", [(True, False), (False, True), (False, False)])
@pytest.mark.parametrize("m,n,k", [(128, 128, 64), (512, 2048, 8192), (2048, 512, 4096), (8192, 1024, 512),
                                   (136, 72, 200)])
def test_gemm_mn_major(amaj, bmaj, m, n, k):
    from flpr_b200.ops.gemm import gemm
    torch.manual_seed(1)
    a = torch.randn(m, k, device="cuda")
    b = torch.randn(n, k, device="cuda")
    ref = _ref_gemm(a, b)
    aa = a.bfloat16() if amaj else a.t().contiguous().bfloat16()
    bb = b.bfloat16() if bmaj else b.t().contiguous().bfloat16()
    out = gemm(aa, bb, a_kmajor=amaj, b_kmajor=bmaj, out_dtype=torch.float32)
    _close(out, ref, rtol=1e-3, atol=1e-3 * math.sqrt(k))


def test_gemm_epilogues():
    from flpr_b200.ops.gemm import gemm
    torch.manual_seed(2)
    m, n, k = 300, 520, 256
    a = torch.randn(m, k, device="cuda").bfloat16()
    b = torch.randn(n, k, device="cuda").bfloat16()
    bias_n = torch.randn(n, device="cuda")
    bias_m = torch.randn(m, device="cuda")
    res = torch.randn(m, n, device="cuda").bfloat16()
    ref = 0.5 * (a.float() @ b.float().t()) + bias_n[None] + bias_m[:, None] + res.float()
    out = gemm(a, b, out_dtype=torch.float32, alpha=0.5, bias_n=bias_n, bias_m=bias_m, residual=res)
    _close(out, ref, rtol=1e-3, atol=2e-2)
    out = gemm(a, b, out_dtype=torch.bfloat16, alpha=0.5, bias_n=bias_n, bias_m=bias_m, residual=res, relu=True)
    _close(out, torch.relu(ref))
    # transposed output (swap-AB style)
    out_t = gemm(a, b, out_dtype=torch.float32, trans_out=True)
    _close(out_t, (a.float() @ b.float().t()).t(), rtol=1e-3, atol=2e-2)
    # split-K
    k2 = 4096
    a2 = torch.randn(256, k2, device="cuda").bfloat16()
    b2 = torch.randn(384, k2, device="cuda").bfloat16()
    out = gemm(a2, b2, out_dtype=torch.float32, split_k=8)
    _close(out, a2.float() @ b2.float().t(), rtol=1e-3, atol=0.1)


@pytest.mark.parametrize("n,h,w,c,cout", [(4, 16, 8, 512, 512), (3, 8, 4, 64, 128), (2, 32, 16, 128, 64),
                                          (5, 16, 8, 64, 96), (8, 8, 4, 128, 256)])
@pytest.mark.parametrize("ks", [1, 3])
def test_conv_nhwc(n, h, w, c, cout, ks):
    from flpr_b200.ops.gemm import conv_nhwc
    torch.manual_seed(3)
    x = torch.randn(n, h, w, c, device="cuda").bfloat16()
    wt = (torch.randn(cout, ks, ks, c, device="cuda") / math.sqrt(c * ks * ks)).bfloat16()
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), wt.float().permute(0, 3, 1, 2),
                                     padding=ks // 2).permute(0, 2, 3, 1)
    out = conv_nhwc(x, wt, padding=ks // 2, out_dtype=torch.float32)
    _close(out, ref, rtol=1e-3, atol=2e-2)


@pytest.mark.parametrize("n,h,w,cin,cout", [(4, 16, 8, 512, 512), (3, 8, 4, 64, 128), (2, 32, 16, 128, 64),
                                            (64, 16, 8, 512, 512)])
@pytest.mark.parametrize("bn", [0, 64, 128, 256])
def test_conv_dgrad_from_forward_weight(n, h, w, cin, cout, bn):
    """dgrad straight from the forward weight (mirrored taps, MN-major B operand) vs conv2d_input."""
    from flpr_b200.ops.gemm import conv_dgrad_nhwc
    if bn > cin:
        pytest.skip("tile wider than N")
    torch.manual_seed(31)
    dy = torch.randn(n, h, w, cout, device="cuda").bfloat16()
    wt = (torch.randn(cout, 3, 3, cin, device="cuda") / math.sqrt(cout * 9)).bfloat16()
    ref = torch.nn.grad.conv2d_input((n, cin, h, w), wt.float().permute(0, 3, 1, 2), dy.float().permute(0, 3, 1, 2),
                                     padding=1).permute(0, 2, 3, 1)
    out = conv_dgrad_nhwc(dy, wt, padding=1, out_dtype=torch.float32, bn=bn)
    _close(out, ref, rtol=1e-3, atol=2e-2)


@pytest.mark.parametrize("m,n,k", [(8192, 512, 1024), (8192, 2048, 512), (200, 136, 320), (1000, 2048, 256)])
@pytest.mark.parametrize("bn", [0, 128, 256])
def test_gemm_fused_bn_statistics(m, n, k, bn):
    """col_part epilogue: 32-row partial column sums / sums of squares of the fp32 result."""
    from flpr_b200.ops.gemm import gemm, col_part_buffer
    torch.manual_seed(32)
    a = torch.randn(m, k, device="cuda").bfloat16()
    b = (torch.randn(n, k, device="cuda") / math.sqrt(k)).bfloat16()
    part = col_part_buffer(m, n, "cuda")
    part.fill_(float("nan"))
    y = gemm(a, b, col_part=part, bn=bn)
    ref = a.float() @ b.float().t()
    _close(y, ref)
    assert torch.isfinite(part).all()
    # the statistics are those of the stored (bf16-rounded) output, accumulated in fp32
    yf = y.float()
    _close(part[:, 0].sum(0), yf.sum(0), rtol=1e-4, atol=1e-3 * yf.abs().sum(0).max().item())
    _close(part[:, 1].sum(0), (yf * yf).sum(0), rtol=1e-4, atol=1e-3 * (yf * yf).sum(0).max().item())
    _close(part[0, 0], yf[:32].sum(0), rtol=1e-4, atol=1e-3)                   # first partial row = rows 0..31
    _close(part[:, 0].sum(0), ref.sum(0), rtol=2e-2, atol=2e-2 * ref.abs().sum(0).max().item())


def test_conv_bn_fused_statistics_match_unfused():
    """conv(+stats in the epilogue) -> BN must equal conv -> BN(with its own statistics pass), fwd and bwd."""
    from flpr_b200.ops.gemm import conv3x3, linear
    from flpr_b200.ops.fused import batch_norm_nhwc
    torch.manual_seed(33)
    for kind in ("conv", "linear"):
        outs = []
        for fused in (True, False):
            torch.manual_seed(34)
            if kind == "conv":
                x = torch.randn(16, 16, 8, 128, device="cuda").bfloat16().requires_grad_(True)
                w = (torch.randn(256, 3, 3, 128, device="cuda") / 30).requires_grad_(True)
            else:
                x = torch.randn(2048, 512, device="cuda").bfloat16().requires_grad_(True)
                w = (torch.randn(256, 512, device="cuda") / 20).requires_grad_(True)
            g = torch.rand(256, device="cuda").add_(0.5).requires_grad_(True)
            b = torch.randn(256, device="cuda").requires_grad_(True)
            rm, rv = torch.zeros(256, device="cuda"), torch.ones(256, device="cuda")
            fn = conv3x3 if kind == "conv" else linear
            if fused:
                y, part = fn(x, w, None, None, True)
            else:
                y, part = fn(x, w), None
            # relu=False: a ReLU mask flips on bf16-level differences of near-zero outputs and would dominate the
            # comparison of the gradients
            z = batch_norm_nhwc(y.reshape(-1, 256), g, b, rm, rv, training=True, relu=False, pre_part=part)
            gz = torch.randn(z.shape, device="cuda", generator=torch.Generator("cuda").manual_seed(5)).bfloat16()
            z.backward(gz)
            outs.append((z.detach(), x.grad, w.grad, g.grad, b.grad, rm, rv))
        for a_, b_ in zip(*outs):
            # statistics from fp32 accumulators vs from the bf16-rounded activation: bf16-level differences
            _close(a_, b_, rtol=5e-2, atol=5e-2 * b_.float().abs().max().item() + 1e-6)


def test_linear_and_conv_autograd():
    from flpr_b200.ops.gemm import linear, conv3x3
    torch.manual_seed(4)
    x = torch.randn(256, 512, device="cuda").bfloat16().requires_grad_(True)
    w = (torch.randn(384, 512, device="cuda") / 20).requires_grad_(True)
    y = linear(x, w)
    gy = torch.randn_like(y)
    y.backward(gy)
    xr = x.detach().float().requires_grad_(True)
    wr = w.detach().bfloat16().float().requires_grad_(True)
    yr = xr @ wr.t()
    yr.backward(gy.float())
    _close(y, yr)
    _close(x.grad, xr.grad)
    _close(w.grad, wr.grad, rtol=1e-2, atol=0.05 * wr.grad.abs().max().item())

    xc = torch.randn(4, 16, 8, 128, device="cuda").bfloat16().requires_grad_(True)
    wc = (torch.randn(64, 3, 3, 128, device="cuda") / 30).requires_grad_(True)
    yc = conv3x3(xc, wc)
    gc = torch.randn_like(yc)
    yc.backward(gc)
    xr = xc.detach().float().permute(0, 3, 1, 2).requires_grad_(True)
    wr = wc.detach().bfloat16().float().permute(0, 3, 1, 2).requires_grad_(True)
    yr = torch.nn.functional.conv2d(xr, wr, padding=1)
    yr.backward(gc.float().permute(0, 3, 1, 2))
    _close(yc, yr.permute(0, 2, 3, 1))
    _close(xc.grad, xr.grad.permute(0, 2, 3, 1))
    _close(wc.grad, wr.grad.permute(0, 2, 3, 1), rtol=1e-2, atol=0.05 * wr.grad.abs().max().item())


@pytest.mark.parametrize("kind", ["adam", "sgd"])
def test_fused_optimizer(kind):
    from flpr_b200.ops.fused import fused_optimizer_step
    torch.manual_seed(5)
    n = 1 << 20
    dev = "cuda"

    def mk():
        torch.manual_seed(5)
        return [torch.randn(n), torch.randn(n), torch.zeros(n), torch.zeros(n), torch.rand(n), torch.randn(n),
                torch.randn(n)]
    cpu = mk()
    gpu = [t.to(dev) for t in mk()]
    st_c, st_g = torch.zeros(2), torch.zeros(2, device=dev)
    shadow = torch.empty(n, dtype=torch.bfloat16, device=dev)
    for step in (1, 2, 3):
        for (p, g, m, v, Q, R, G), st, sh in ((cpu, st_c, None), (gpu, st_g, shadow)):
            fused_optimizer_step(kind, p, g, m, v, lr=1e-3, step=step, weight_decay=1e-5, momentum=0.9, Q=Q, R=R,
                                 lam2=0.3, G=G, lam1=1e-3, atten=0.9, p_bf16=sh, stats=st)
    _close(gpu[0].cpu(), cpu[0], rtol=1e-4, atol=1e-5)
    _close(gpu[2].cpu(), cpu[2], rtol=1e-4, atol=1e-5)
    _close(st_g.cpu(), st_c, rtol=1e-3, atol=1.0)
    _close(shadow.float().cpu(), cpu[0], rtol=1e-2, atol=1e-2)


@pytest.mark.parametrize("kind", ["adam", "sgd"])
def test_fused_trained_l1_anchor(kind):
    """FedSTIL's trained L1 anchor inside ``fused_opt_kernel`` (reference quirk, fedstil.py:53-76,639-647) against the
    fp32 tensor-op form on the CPU (``ArenaOptimizer._anchor_step``, the one the golden tests compare with the
    reference) over several steps: weights, anchor, both moment pairs, the bf16 shadow and the reported L1 sum."""
    import torch.nn as nn
    from flpr_b200.runtime.arena import ArenaOptimizer, ParamArena
    outs = {}
    for dev in ("cpu", "cuda"):
        torch.manual_seed(11)
        lin1, lin2 = nn.Linear(256, 512, bias=False), nn.Linear(512, 64)
        params = [("a.weight", lin1.weight), ("b.weight", lin2.weight), ("b.bias", lin2.bias)]
        arena = ParamArena(params, dev, shadow=dev == "cuda", first=lambda n: n == "a.weight")
        opt = ArenaOptimizer(kind, arena, lr=1e-3 if kind == "adam" else 0.05, weight_decay=1e-4, momentum=0.9)
        n = arena.prefix_numel
        torch.manual_seed(12)
        G = (arena.master[:n].cpu() + 0.01 * torch.randn(n)).to(dev)
        opt.G, opt.lam1, opt.atten = G, 1e-2, 0.9
        opt.anchor = G.clone()
        opt.stats = torch.zeros(2, device=dev)
        for step in range(4):
            torch.manual_seed(100 + step)
            g = torch.randn(arena.numel) * (torch.rand(arena.numel) > 0.3)     # exact zeros: the sign(0) = 0 rule
            arena.grad.copy_(g.to(dev))
            opt.step()
        outs[dev] = [arena.master.cpu(), opt.anchor.cpu(), opt.m.cpu(),
                     opt.anchor_m.cpu() if opt.anchor_m is not None else torch.zeros(1), opt.stats.cpu(),
                     arena.shadow.float().cpu() if arena.shadow is not None else None]
        if dev == "cuda":
            assert opt.anchor_m is not None                      # the fused path allocated the anchor's moments
    c, g = outs["cpu"], outs["cuda"]
    _close(g[0], c[0], rtol=1e-4, atol=2e-6)
    _close(g[1], c[1], rtol=1e-4, atol=2e-6)
    _close(g[2], c[2], rtol=1e-3, atol=1e-5)
    _close(g[3], c[3], rtol=1e-3, atol=1e-6)
    _close(g[4][1:], c[4][1:], rtol=1e-3, atol=1e-2)
    _close(g[5], c[0], rtol=1e-2, atol=1e-2)
    assert (c[1] - G.cpu()).abs().max() > 1e-5                   # the anchor did move


def test_importance_and_cast_and_compose():
    from flpr_b200.ops.fused import importance_accumulate, cast_bf16, compose_adaptive
    n = 4096 * 33
    g = torch.randn(n, device="cuda")
    F1 = torch.zeros(n, device="cuda")
    importance_accumulate(F1, g, 0.25, "fisher")
    importance_accumulate(F1, g, 0.5, "mas")
    _close(F1, 0.25 * g * g + 0.5 * g.abs(), rtol=1e-5, atol=1e-6)
    _close(cast_bf16(g), g.bfloat16().float(), rtol=0, atol=0)
    G = torch.randn(n, device="cuda")
    A = torch.randn(n, device="cuda")
    th = torch.empty(n, device="cuda")
    thb = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    compose_adaptive(G, A, 0.9, th, thb)
    _close(th, 0.9 * G + A, rtol=1e-6, atol=1e-6)
    _close(thb, (0.9 * G + A).bfloat16(), rtol=1e-2, atol=1e-2)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_ce_label_smooth(dtype):
    from flpr_b200.ops.fused import ce_label_smooth, ce_label_smooth_reference
    torch.manual_seed(6)
    b, c = 64, 8000
    logits = (torch.randn(b, c, device="cuda") * 3).to(dtype).requires_grad_(True)
    tgt = torch.randint(0, c, (b,), device="cuda")
    stats = torch.zeros(2, device="cuda")
    loss = ce_label_smooth(logits, tgt, 0.1, stats)
    loss.backward()
    lr = logits.detach().float().requires_grad_(True)
    ref = ce_label_smooth_reference(lr, tgt, 0.1)
    ref.backward()
    assert abs(loss.item() - ref.item()) < 2e-3 * abs(ref.item())
    _close(logits.grad, lr.grad, rtol=2e-2, atol=2e-5)
    assert int(stats[1].item()) == int((lr.argmax(1) == tgt).sum().item())


@pytest.mark.parametrize("relu,res", [(False, False), (True, False), (True, True)])
def test_batch_norm_nhwc(relu, res):
    from flpr_b200.ops.fused import batch_norm_nhwc
    torch.manual_seed(7)
    m, c = 4096, 512
    x = (torch.randn(m, c, device="cuda") * 2 + 0.5).bfloat16().requires_grad_(True)
    r = torch.randn(m, c, device="cuda").bfloat16().requires_grad_(True) if res else None
    gamma = (torch.rand(c, device="cuda") + 0.5).requires_grad_(True)
    beta = torch.randn(c, device="cuda").requires_grad_(True)
    rm, rv = torch.zeros(c, device="cuda"), torch.ones(c, device="cuda")
    y = batch_norm_nhwc(x, gamma, beta, rm, rv, training=True, relu=relu, residual=r)
    gy = torch.randn_like(y)
    y.backward(gy)
    xr = x.detach().float().requires_grad_(True)
    rr = r.detach().float().requires_grad_(True) if res else None
    gr, br = gamma.detach().clone().requires_grad_(True), beta.detach().clone().requires_grad_(True)
    rm2, rv2 = torch.zeros(c, device="cuda"), torch.ones(c, device="cuda")
    yr = torch.nn.functional.batch_norm(xr, rm2, rv2, gr, br, training=True, momentum=0.1, eps=1e-5)
    if res:
        yr = yr + rr
    if relu:
        yr = torch.relu(yr)
    yr.backward(gy.float())
    _close(y, yr, rtol=2e-2, atol=3e-2)
    _close(x.grad, xr.grad, rtol=5e-2, atol=3e-2)
    _close(gamma.grad, gr.grad, rtol=2e-2, atol=0.02 * gr.grad.abs().max().item())
    _close(beta.grad, br.grad, rtol=2e-2, atol=0.02 * br.grad.abs().max().item())
    _close(rm, rm2, rtol=1e-3, atol=1e-3)
    _close(rv, rv2, rtol=1e-3, atol=1e-3)
    if res:
        _close(r.grad, rr.grad, rtol=2e-2, atol=2e-2)


@pytest.mark.parametrize("n,h,w,cin,cout", [(64, 16, 8, 512, 512), (4, 8, 4, 64, 128), (6, 16, 8, 128, 64), (3, 32, 16, 64, 64)])
def test_conv3x3_wgrad_kernel(n, h, w, cin, cout):
    from flpr_b200.ops.gemm import conv3x3_wgrad
    torch.manual_seed(11)
    x = torch.randn(n, h, w, cin, device="cuda").bfloat16()
    dy = (torch.randn(n, h, w, cout, device="cuda") / 8).bfloat16()
    ref = torch.nn.grad.conv2d_weight(x.float().permute(0, 3, 1, 2), (cout, cin, 3, 3), dy.float().permute(0, 3, 1, 2),
                                      padding=1).permute(0, 2, 3, 1)
    out = conv3x3_wgrad(x, dy)
    _close(out, ref, rtol=1e-2, atol=0.02 * ref.abs().max().item())
    slot = torch.zeros(cout, 3, 3, cin, device="cuda")
    conv3x3_wgrad(x, dy, out=slot)
    _close(slot, ref, rtol=1e-2, atol=0.02 * ref.abs().max().item())


@pytest.mark.parametrize("m,c", [(64, 2048), (8192, 512), (1000, 96), (37, 64)])
def test_batch_norm_shapes(m, c):
    from flpr_b200.ops.fused import batch_norm_nhwc
    torch.manual_seed(12)
    x = (torch.randn(m, c, device="cuda") * 1.5 - 0.3).bfloat16().requires_grad_(True)
    gamma = (torch.rand(c, device="cuda") + 0.5).requires_grad_(True)
    beta = torch.randn(c, device="cuda").requires_grad_(True)
    y = batch_norm_nhwc(x, gamma, beta, None, None, training=True, relu=True)
    gy = torch.randn_like(y)
    y.backward(gy)
    xr = x.detach().float().requires_grad_(True)
    gr, br = gamma.detach().clone().requires_grad_(True), beta.detach().clone().requires_grad_(True)
    yr = torch.relu(torch.nn.functional.batch_norm(xr, None, None, gr, br, training=True))
    yr.backward(gy.float())
    _close(y, yr, rtol=2e-2, atol=3e-2)
    _close(x.grad, xr.grad, rtol=5e-2, atol=0.03 * xr.grad.abs().max().item() + 1e-3)
    _close(gamma.grad, gr.grad, rtol=2e-2, atol=0.02 * gr.grad.abs().max().item())


def test_gap():
    from flpr_b200.ops.fused import global_avg_pool_nhwc
    x = torch.randn(16, 128, 2048, device="cuda").bfloat16().requires_grad_(True)
    y = global_avg_pool_nhwc(x)
    y.backward(torch.ones_like(y))
    _close(y, x.float().mean(1), rtol=1e-3, atol=1e-3)
    _close(x.grad, torch.full_like(x, 1 / 128.0).float(), rtol=1e-2, atol=1e-4)


def test_rank_eval():
    from flpr_b200.ops.rank import rank_metrics, rank_metrics_reference, similarity
    torch.manual_seed(8)
    q = torch.nn.functional.normalize(torch.randn(300, 2048, device="cuda"), dim=1)
    g = torch.nn.functional.normalize(torch.randn(1500, 2048, device="cuda"), dim=1)
    ql = torch.randint(0, 60, (300,))
    gl = torch.randint(0, 70, (1500,))
    sim = similarity(q, g, precise=True)
    _close(sim, q @ g.t(), rtol=1e-4, atol=2e-5)
    cmc, m_ap = rank_metrics(sim, ql, gl)
    cmc_r, map_r = rank_metrics_reference(sim.cpu(), ql, gl)
    assert abs(m_ap - map_r) < 1e-5
    assert abs(cmc - cmc_r).max() < 1e-9


def test_comm_single_rank():
    """world_size == 1: the peer kernels degenerate to local HBM traffic but run the same code."""
    from flpr_b200.parallel.comm import FedComm
    K, n = 8, 4096 * 5
    comm = FedComm("cuda", K, arena_bytes=64 << 20)
    comm.alloc_client_buffer("up", n)
    comm.alloc_client_buffer("cnt", 4)
    comm.alloc_client_buffer("fisher", n)
    comm.alloc_rank_buffer("glob", n)
    for nm in ("f", "fp", "fpp"):
        comm.alloc_rank_buffer(nm, n)
    ups, cnts, fis = [], [], []
    for c in range(K):
        u = torch.randn(n, device="cuda")
        comm.client_view("up", c).copy_(u)
        comm.client_view("cnt", c).fill_(float(10 + c))
        f = torch.rand(n, device="cuda")
        comm.client_view("fisher", c).copy_(f)
        ups.append(u); cnts.append(10.0 + c); fis.append(f)
    U = torch.stack(ups)
    w = torch.tensor(cnts, device="cuda"); w = w / w.sum()
    comm.reduce_bcast("up", "glob", list(range(K)), cnt="cnt")
    _close(comm.rank_view("glob"), (w[:, None] * U).sum(0), rtol=1e-5, atol=1e-5)
    rows = torch.softmax(torch.randn(K, K), dim=1)
    outs_g = [torch.empty(n, device="cuda") for _ in range(K)]
    outs_t = [torch.empty(n, device="cuda") for _ in range(K)]
    outs_b = [torch.empty(n, device="cuda", dtype=torch.bfloat16) for _ in range(K)]
    comm.mix("up", list(range(K)), rows, list(range(K)), outs_g, outs_t, outs_b)
    ref = rows.cuda() @ U
    for i in range(K):
        _close(outs_g[i], ref[i], rtol=1e-5, atol=1e-5)
        _close(outs_t[i], ref[i], rtol=1e-5, atol=1e-5)
        _close(outs_b[i], ref[i], rtol=1e-2, atol=2e-2)
    comm.curv_moments("fisher", "up", list(range(K)), "f", "fp", "fpp")
    Fs = torch.stack(fis)
    _close(comm.rank_view("f"), Fs.sum(0), rtol=1e-5, atol=1e-5)
    _close(comm.rank_view("fp"), (Fs * U).sum(0), rtol=1e-5, atol=1e-4)
    _close(comm.rank_view("fpp"), (Fs * U * U).sum(0), rtol=1e-5, atol=1e-4)
    out = torch.empty(n, K, device="cuda")
    comm.gather_strided("up", list(range(K)), out)
    _close(out, U.t(), rtol=0, atol=0)
    d = torch.empty(n, device="cuda"); db = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    comm.pull("up", 3, d, db)
    _close(d, U[3], rtol=0, atol=0)
    comm.barrier()
    torch.cuda.synchronize()
    comm.check_errors()
    comm.close()


@pytest.mark.parametrize("level", ["none", "default", "drastic"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_fused_augmentation_kernel(level, dtype):
    """uint8 NHWC -> normalise + flip + erase + cast in one kernel vs the tensor-op reference (same uniforms)."""
    from flpr_b200.data.augmentation import DeviceAugment
    aug = DeviceAugment(level, dtype=dtype)
    u8 = torch.randint(0, 256, (37, 256, 128, 3), dtype=torch.uint8, device="cuda")
    g = torch.Generator("cuda")
    g.manual_seed(7)
    out = aug(u8, g)
    g.manual_seed(7)
    ref = aug.reference(u8, g)
    assert out.shape == ref.shape == (37, 3, 256, 128) and out.dtype == dtype
    assert out.is_contiguous(memory_format=torch.channels_last)
    tol = 2e-2 if dtype == torch.bfloat16 else 1e-5
    # a rounding difference in the rectangle size may move an edge by one pixel on a few samples
    bad = ((out.float() - ref.float()).abs() > tol).flatten(1).any(1).sum().item()
    assert bad <= 2, f"{bad} samples differ"


def test_herding_kernel_matches_tensor_path():
    from flpr_b200.methods.fedstil import herding_select, herding_select_batched, group_matrix
    torch.manual_seed(11)
    feats = torch.randn(300, 2048, device="cuda")
    sizes = [1, 5, 8, 17, 64, 40]
    groups, o = [], 0
    perm = torch.randperm(300, device="cuda")
    for n in sizes:
        groups.append(perm[o:o + n])
        o += n
    idx, counts = group_matrix(groups)
    picks = herding_select_batched(feats, idx, counts, 12).cpu()
    for gi, g in enumerate(groups):
        ref = herding_select(feats[g].cpu(), 12)
        assert picks[gi].tolist() == ref, (gi, picks[gi].tolist(), ref)


def test_bulk_device_loader_covers_split():
    from flpr_b200.data.synthetic import random_array_split
    from flpr_b200.data.pipeline import DeviceBatchLoader
    ds = random_array_split(100, 10, (64, 32), seed=3)
    ld = DeviceBatchLoader(ds, 32, shuffle=True, level="none", mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225),
                           device="cuda", dtype=torch.float32, seed=1)
    assert ld._bulk_ok()
    seen, n = [], 0
    for data, pid, cid in ld:
        assert data.is_cuda and data.shape[1:] == (3, 64, 32)
        n += data.shape[0]
        seen.append(pid)
    assert n == 100 and sorted(torch.cat(seen).tolist()) == sorted(ds.pids.tolist())
    wide = [d.shape[0] for d, _, _ in ld.iterate(64, ordered=True)]
    assert wide == [64, 36]
    ref = ld.augment.reference(ds.images[:64].cuda())
    first = next(iter(ld.iterate(64, ordered=True)))[0]
    assert torch.allclose(first, ref, atol=1e-5)
    assert ld.h2d_bytes >= 2 * ds.images.numel()


@pytest.mark.parametrize("n,h,w,c,cout,ks", [(4, 64, 32, 128, 128, 3), (3, 32, 16, 256, 256, 3), (4, 64, 32, 256, 512, 1),
                                             (2, 32, 16, 512, 1024, 1), (5, 16, 8, 64, 64, 3)])
def test_strided_conv_via_tma_element_strides(n, h, w, c, cout, ks):
    """Stride-2 convolution = the same implicit-GEMM pipeline over a tensor map with element strides {1,2,2,1}."""
    from flpr_b200.ops.gemm import conv_nhwc
    torch.manual_seed(41)
    x = torch.randn(n, h, w, c, device="cuda").bfloat16()
    wt = (torch.randn(cout, ks, ks, c, device="cuda") / math.sqrt(c * ks * ks)).bfloat16()
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), wt.float().permute(0, 3, 1, 2), padding=ks // 2,
                                     stride=2).permute(0, 2, 3, 1)
    out = conv_nhwc(x, wt, padding=ks // 2, stride=2, out_dtype=torch.float32)
    assert out.shape == ref.shape
    _close(out, ref, rtol=1e-3, atol=2e-2)


@pytest.mark.parametrize("m,n,k", [(8192, 256, 64), (4096, 64, 256), (1000, 2048, 512)])
def test_lean_epilogue_bias_residual_relu(m, n, k):
    """Inference epilogue of the folded trunk: bf16( relu( A B^T + bias[col] + residual ) ) on the lean path."""
    from flpr_b200.ops.gemm import gemm, conv_nhwc
    torch.manual_seed(42)
    a = torch.randn(m, k, device="cuda").bfloat16()
    b = (torch.randn(n, k, device="cuda") / math.sqrt(k)).bfloat16()
    bias = torch.randn(n, device="cuda")
    res = torch.randn(m, n, device="cuda").bfloat16()
    ref = a.float() @ b.float().t() + bias[None]
    _close(gemm(a, b, bias_n=bias, relu=True), torch.relu(ref))
    _close(gemm(a, b, bias_n=bias, relu=True, residual=res), torch.relu(ref + res.float()))
    _close(gemm(a, b, bias_n=bias), ref)
    x = torch.randn(8, 16, 8, 128, device="cuda").bfloat16()
    wt = (torch.randn(256, 3, 3, 128, device="cuda") / 34).bfloat16()
    bias = torch.randn(256, device="cuda")
    res = torch.randn(8, 16, 8, 256, device="cuda").bfloat16()
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), wt.float().permute(0, 3, 1, 2),
                                     padding=1).permute(0, 2, 3, 1) + bias
    _close(conv_nhwc(x, wt, padding=1, bias=bias, relu=True, residual=res), torch.relu(ref + res.float()))


@pytest.mark.parametrize("b,h,w", [(16, 256, 128), (8, 128, 64), (3, 64, 32)])
def test_native_stem_and_maxpool(b, h, w):
    """7x7/2 stem as a 4x4 conv over space-to-depth cells (overlapping TMA windows) + NHWC max-pool."""
    from flpr_b200.ops.gemm import stem_weight_s2d, stem_conv, maxpool3x3s2, s2d_pad
    torch.manual_seed(51)
    x = torch.randn(b, h, w, 3, device="cuda").bfloat16()
    wt = (torch.randn(64, 3, 7, 7, device="cuda") / 12).bfloat16().float()
    bias = torch.randn(64, device="cuda")
    cells = s2d_pad(x)
    assert torch.equal(cells.cpu(), s2d_pad(x.cpu()))
    ref = torch.relu(torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), wt, bias, stride=2, padding=3))
    out = stem_conv(x, stem_weight_s2d(wt).bfloat16(), bias)
    _close(out, ref.permute(0, 2, 3, 1))
    pooled = maxpool3x3s2(out)
    refp = torch.nn.functional.max_pool2d(out.float().permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    assert torch.equal(pooled.float(), refp)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("bw,n,h,d,nwb", [(8, 49, 3, 32, 1), (16, 49, 6, 32, 4), (4, 16, 24, 32, 1), (6, 49, 12, 64, 2)])
def test_fused_window_attention(dtype, bw, n, h, d, nwb):
    """Swin window attention in one kernel (fwd + bwd) vs the tensor-op reference in fp32."""
    from flpr_b200.ops.fused import window_attention
    torch.manual_seed(61)
    qkv = torch.randn(bw, n, 3, h, d, device="cuda").to(dtype).requires_grad_(True)
    bias = (torch.randn(nwb, h, n, n, device="cuda") * 0.5).requires_grad_(True)
    scale = d ** -0.5
    out = window_attention(qkv, bias, scale)
    g = torch.randn_like(out)
    out.backward(g)
    q32 = qkv.detach().float().requires_grad_(True)
    b32 = bias.detach().clone().requires_grad_(True)
    q, k, v = q32.permute(2, 0, 3, 1, 4)
    s = (q * scale) @ k.transpose(-1, -2)
    s = s.view(bw // nwb, nwb, h, n, n) + b32.unsqueeze(0)
    ref = (torch.softmax(s.view(bw, h, n, n), -1) @ v).transpose(1, 2).reshape(bw, n, h * d)
    ref.backward(g.float())
    tol = 3e-2 if dtype == torch.bfloat16 else 1e-4
    _close(out, ref, rtol=tol, atol=tol * ref.abs().max().item())
    _close(qkv.grad, q32.grad, rtol=tol, atol=tol * q32.grad.abs().max().item())
    _close(bias.grad, b32.grad, rtol=tol, atol=tol * b32.grad.abs().max().item() + 1e-6)


@pytest.mark.parametrize("cosine", [False, True])
@pytest.mark.parametrize("hard", [False, True])
@pytest.mark.parametrize("margin", [0.3, None])
def test_fused_triplet_loss_matches_tensor_ops(cosine, hard, margin):
    """Triplet loss with the Gram matrix on the wgmma GEMM and fused mining (``csrc/loss_ops.cu``), forward and the
    gradient w.r.t. the features, against the plain fp32 tensor-op form (``criterions/triplet_loss.py:89-127``)."""
    from flpr_b200.criterions import TripletLoss
    torch.manual_seed(3)
    b, d = 64, 2048
    labels = torch.arange(16, device="cuda").repeat_interleave(4)[torch.randperm(b, device="cuda")]
    x0 = (torch.randn(b, d, device="cuda") * 0.5 + labels[:, None].float() * 0.01)
    outs = []
    for fused in (True, False):
        x = x0.clone().requires_grad_(True)
        crit = TripletLoss(margin=margin, norm_feat=cosine, hard_mining=hard)
        crit.fused = fused
        loss = crit(feature=x, target=labels)
        loss.backward()
        outs.append((loss.detach(), x.grad.detach()))
    (lf, gf), (lr, gr) = outs
    assert abs(lf.item() - lr.item()) <= 2e-3 * max(1.0, abs(lr.item())), (lf.item(), lr.item())
    cos = torch.nn.functional.cosine_similarity(gf.flatten(), gr.flatten(), dim=0).item()
    assert cos > 0.999, cos
    assert (gf - gr).abs().max().item() <= 2e-2 * gr.abs().max().item() + 1e-7


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_fused_kd_and_bce_distill(dtype):
    import torch.nn.functional as F
    from flpr_b200.ops.fused import bce_distill, kd_kl
    torch.manual_seed(5)
    b, c, p = 48, 730, 500
    s0 = (torch.randn(b, c, device="cuda") * 2).to(dtype)
    t = (torch.randn(b, c, device="cuda") * 2).to(dtype)
    s = s0.clone().requires_grad_(True)
    T = 4.0
    loss = kd_kl(s, t, T)
    loss.backward()
    sr = s0.float().clone().requires_grad_(True)
    ref = F.kl_div(F.log_softmax(sr / T, dim=1), F.softmax(t.float() / T, dim=1), reduction="sum") * T * T / b
    ref.backward()
    assert abs(loss.item() - ref.item()) < 2e-3 * max(1.0, abs(ref.item()))
    _close(s.grad.float(), sr.grad, rtol=2e-2, atol=2e-2 * sr.grad.abs().max().item())
    # iCaRL distillation pass
    tgt = torch.randint(0, c, (b,), device="cuda")
    prev = torch.randn(b, p, device="cuda")
    z = s0.clone().requires_grad_(True)
    l2 = bce_distill(z, tgt, prev)
    l2.backward()
    zr = s0.float().clone().requires_grad_(True)
    onehot = torch.zeros(b, c, device="cuda").scatter_(1, tgt.view(-1, 1), 1.0)
    r2 = F.binary_cross_entropy_with_logits(zr, onehot) + F.binary_cross_entropy_with_logits(zr[:, :p], torch.sigmoid(prev))
    r2.backward()
    assert abs(l2.item() - r2.item()) < 2e-3 * max(1.0, abs(r2.item()))
    _close(z.grad.float(), zr.grad, rtol=2e-2, atol=2e-2 * zr.grad.abs().max().item())


@pytest.mark.parametrize("bw,n,h,nwb", [(64 * 64, 49, 3, 64), (64 * 16, 49, 6, 16), (64, 49, 24, 1), (37, 16, 12, 1)])
def test_window_attention_tcgen05_forward(bw, n, h, nwb):
    """(Name kept from the Blackwell version of the kernel.) The wgmma forward (QK^T and PV on the tensor cores, register accumulators, quad-per-row softmax) against the
    CUDA-core kernel and the fp32 tensor-op reference, at the real Swin-T stage shapes (batch 64)."""
    from flpr_b200.ops import native
    from flpr_b200.ops.fused import window_attention
    lib = native.load()
    torch.manual_seed(7)
    d = 32
    qkv = torch.randn(bw, n, 3, h, d, device="cuda").to(torch.bfloat16)
    bias = torch.randn(nwb, h, n, n, device="cuda") * 0.5
    bias[:, :, :, -3:] -= 100.0 * (torch.rand(nwb, h, n, 3, device="cuda") > 0.7)       # shift-mask like entries
    scale = d ** -0.5
    outs = {}
    for tc in (1, 0):
        lib.flpr_window_attn_set_tc(tc)
        with torch.no_grad():
            outs[tc] = window_attention(qkv, bias, scale).float()
    lib.flpr_window_attn_set_tc(1)
    q, k, v = qkv.float().permute(2, 0, 3, 1, 4)
    s = (q * scale) @ k.transpose(-1, -2)
    s = s.view(bw // nwb, nwb, h, n, n) + bias.unsqueeze(0)
    ref = (torch.softmax(s.view(bw, h, n, n), -1) @ v).transpose(1, 2).reshape(bw, n, h * d)
    _close(outs[1], ref, rtol=3e-2, atol=3e-2 * ref.abs().max().item())
    _close(outs[1], outs[0], rtol=3e-2, atol=3e-2 * ref.abs().max().item())

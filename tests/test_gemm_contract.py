"""The wgmma GEMM / implicit-GEMM convolution family (``csrc/gemm_wgmma.cu``) against a float64 oracle, across its
argument contract: operand-major combinations, K / M / N edges, strided operands and outputs, every epilogue option,
fused batch-norm statistics, split-K and the convolution entry points.

Every element is compared against a bound that scales with that element's own magnitude (:func:`assert_within`), on
inputs whose rows and columns are scaled by powers of two from 2^-10 to 2^10: a wrong value in a small-valued tile
cannot hide under the largest element of the output. The CPU reference path of ``ops/gemm.py`` is held to the same
bound on the same inputs, and the option combinations the kernel cannot compute as one result are refused on both
devices.

CPU tests are unmarked. GPU tests carry ``pytest.mark.gpu`` and run under every kernel variant (:func:`gpu`).
"""
import contextlib
import math

import pytest
import torch
import torch.nn.functional as F

from flpr_b200.ops import gemm as gops
from flpr_b200.ops import native

# ------------------------------------------------------------------------------------------------- the bound
# |x - ref| <= C_BOUND * 2^-16 * scale  (+ 2^-8 * |ref| for a bf16 output)  + FLOOR, per element, where
# scale = |alpha| (|A| |B|^T) + |bias_n| + |bias_m| + |residual| in float64, the magnitude the fp32 result is built
# from.
# C_BOUND = 16 makes the first term 2^-12 * scale. The worst-case forward error of a length-K fp32 sum is about
# K * 2^-24 * scale (Higham, "Accuracy and Stability of Numerical Algorithms", 2nd ed., section 3.1), which 2^-12 covers
# for K <= 4096; the tensor cores add the products of one k16 MMA step before they reach the fp32 accumulator, so the
# chain of accumulator roundings is much shorter than K and the longest K here (4104) is covered too. The second term
# is the worst-case round-to-nearest error of bf16 (8 significand bits). The oracle self-test below shows that this
# bound still rejects a dropped K block, a doubled bias, a shifted chunk, truncation instead of rounding and a 1e-3
# relative error in the smallest-valued tile.
C_BOUND = 16
FLOOR = 1e-30


def within(x: torch.Tensor, ref: torch.Tensor, scale: torch.Tensor, bf16_out: bool) -> torch.Tensor:
    """Elementwise: ``x`` (kernel output, any dtype) is within the bound of the float64 ``ref`` (NaN never is)."""
    bound = C_BOUND * 2.0 ** -16 * scale + FLOOR
    if bf16_out:
        bound = bound + 2.0 ** -8 * ref.abs()
    return (x.double() - ref).abs() <= bound


def assert_within(x, ref, scale, bf16_out, what="output"):
    assert x.shape == ref.shape, (what, tuple(x.shape), tuple(ref.shape))
    ok = within(x, ref, scale, bf16_out)
    if not bool(ok.all()):
        bad = (~ok).nonzero()
        i = tuple(bad[0].tolist())
        raise AssertionError(f"{what}: {bad.shape[0]} of {ok.numel()} elements outside the bound; first at {i}: "
                             f"got {x[i].item()!r}, float64 reference {ref[i].item()!r}, scale {scale[i].item()!r}")


def oracle(a, b, *, alpha=1.0, bias_n=None, bias_m=None, residual=None, relu=False, trans_out=False):
    """float64 epilogue(alpha * A @ B^T) and its error scale; ``a`` [M,K], ``b`` [N,K] (already bf16)."""
    A, B = a.double(), b.double()
    d = alpha * (A @ B.t())
    s = abs(alpha) * (A.abs() @ B.abs().t())
    if bias_n is not None:
        d, s = d + bias_n.double()[None], s + bias_n.double().abs()[None]
    if bias_m is not None:
        d, s = d + bias_m.double()[:, None], s + bias_m.double().abs()[:, None]
    if trans_out:
        d, s = d.t(), s.t()
    if residual is not None:
        d, s = d + residual.double(), s + residual.double().abs()
    if relu:
        d = d.clamp_min(0)
    return d, s


def col_part_oracle(stored: torch.Tensor, rows: int):
    """float64 32-row partial sums (and sums of squares) of the stored ``[M, N]`` output; rows past M count as 0."""
    m, n = stored.shape
    y = torch.cat([stored.double(), stored.new_zeros(rows * 32 - m, n, dtype=torch.float64)]).view(rows, 32, n)
    s2 = (y * y).sum(1)
    return y.sum(1), y.abs().sum(1), s2


def assert_col_part(part, stored, m):
    s1, a1, s2 = col_part_oracle(stored, part.shape[0])
    assert_within(part[:, 0], s1, a1, False, "col_part sums")
    assert_within(part[:, 1], s2, s2, False, "col_part sums of squares")
    for r in range(part.shape[0]):
        if r * 32 >= m:                                    # a partial row made only of padding rows
            assert bool((part[r] == 0).all()), f"col_part row {r} (padding only) is not 0"


# ------------------------------------------------------------------------------------------------- inputs
def _pow2(n, g, block=32):
    """2^e per index, e in -10..10: drawn once per ``block`` indices (32 = one epilogue chunk), plus -1..1 per index."""
    e = torch.randint(-10, 11, (-(-n // block),), generator=g).repeat_interleave(block)[:n]
    e = (e + torch.randint(-1, 2, (n,), generator=g)).clamp(-10, 10)
    return torch.exp2(e.double())


def operands(m, n, k, seed):
    """bf16 A [M,K], B [N,K] with row i of A scaled by 2^e_i and row j of B (output column j) by 2^f_j, e and f
    changing every 32 rows / columns, so that neighbouring 32 x 32 output chunks differ in magnitude by orders; plus
    the two scale vectors."""
    g = torch.Generator().manual_seed(seed)
    rs, cs = _pow2(m, g), _pow2(n, g)
    a = (torch.randn(m, k, generator=g, dtype=torch.float64) * rs[:, None]).bfloat16()
    b = (torch.randn(n, k, generator=g, dtype=torch.float64) * cs[:, None]).bfloat16()
    return a, b, rs, cs


def place(t, dev, pad=0, row0=0, fill=float("nan")):
    """``t`` (2-D) as a view into a larger ``fill``-ed buffer on ``dev``: row stride ``round8(cols) + pad``, first row
    ``row0``, first column 8 when ``pad >= 8``. Kept 16-byte aligned, as the TMA operands must be."""
    rows, cols = t.shape
    ld = -(-cols // 8) * 8 + pad
    c0 = 8 if pad >= 8 else 0
    buf = torch.full((row0 + rows, ld), fill, dtype=t.dtype, device=dev)
    v = buf[row0:, c0:c0 + cols]
    v.copy_(t)
    return v


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def out_view(shape, dtype, dev, ld, c0=0):
    """A ``shape`` view with row stride ``ld`` starting at column ``c0`` of a NaN-filled buffer, and the buffer."""
    rows, cols = shape
    buf = torch.full((rows + 1, ld), float("nan"), dtype=dtype, device=dev)
    return buf[:rows, c0:c0 + cols], buf


def assert_outside_untouched(buf, view):
    """Every element of ``buf`` outside ``view`` still holds the NaN it was filled with, bit for bit."""
    nan = _bits(torch.full((1,), float("nan"), dtype=buf.dtype, device=buf.device))
    mask = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    off = view.storage_offset() - buf.storage_offset()
    r0, c0 = divmod(off, buf.stride(0))
    mask[r0:r0 + view.shape[0], c0:c0 + view.shape[1]] = False
    outside = _bits(buf)[mask]
    assert bool((outside == nan).all()), f"{int((outside != nan).sum())} elements outside [M, N] were written"


def gemm_case(dev, m, n, k, *, amaj=True, bmaj=True, out_dtype=torch.float32, alpha=1.0, epi=(), trans_out=False,
              bn=0, split_k=1, pad=0, row0=0, out_ld=None, out_c0=0, prefill=False, bias_offset=0, seed=0):
    """Run ``gops.gemm`` on ``dev`` for one configuration and check every element (and, with ``out_ld``, that nothing
    outside ``[M, N]`` of the output buffer was written). ``epi`` names the epilogue options in use."""
    a, b, rs, cs = operands(m, n, k, seed)
    g = torch.Generator().manual_seed(seed + 1)
    t = math.sqrt(k)
    bias_n = bias_m = res = None
    if "bias_n" in epi:
        bias_n = (torch.randn(n, generator=g, dtype=torch.float64) * cs * t).float().to(dev)
        if bias_offset:                                    # a view that is not 16-byte aligned
            bias_n = torch.cat([bias_n.new_zeros(bias_offset), bias_n])[bias_offset:]
            assert bias_n.data_ptr() % 16 != 0
    if "bias_m" in epi:
        bias_m = (torch.randn(m, generator=g, dtype=torch.float64) * rs * t).float().to(dev)
    oshape = (n, m) if trans_out else (m, n)
    if "residual" in epi:
        r = torch.randn(m, n, generator=g, dtype=torch.float64) * rs[:, None] * cs[None] * t
        res = (r.t() if trans_out else r).bfloat16().contiguous()
    relu = "relu" in epi
    ref, scale = oracle(a.to(dev), b.to(dev), alpha=alpha, bias_n=bias_n, bias_m=bias_m,
                        residual=None if res is None else res.to(dev), relu=relu, trans_out=trans_out)
    aa = place(a if amaj else a.t(), dev, pad, row0)
    bb = place(b if bmaj else b.t(), dev, pad, row0)
    out = buf = None
    if out_ld is not None:
        out, buf = out_view(oshape, out_dtype, dev, out_ld, out_c0)
        if prefill:                                        # garbage the kernel must overwrite, not add to
            out.copy_(torch.randn(oshape, generator=g) * 1e3)
        if res is not None:
            rv, _ = out_view(oshape, torch.bfloat16, dev, out_ld, out_c0)
            rv.copy_(res)
            res = rv
    if res is not None:
        res = res.to(dev)
    y = gops.gemm(aa, bb, a_kmajor=amaj, b_kmajor=bmaj, out_dtype=out_dtype, trans_out=trans_out, alpha=alpha,
                  bias_n=bias_n, bias_m=bias_m, relu=relu, residual=res, split_k=split_k, bn=bn, out=out)
    if out is not None:
        assert y.data_ptr() == out.data_ptr()
        assert_outside_untouched(buf, out)
    assert y.dtype == out_dtype
    assert_within(y, ref, scale, out_dtype == torch.bfloat16)
    return y


# ------------------------------------------------------------------------------------------------- kernel variants
VARIANTS = ("persistent", "classic", "pair", "generic-epilogue")


@contextlib.contextmanager
def kernel_variant_set(name):
    """Persistent grid (default), one CTA per tile, the CTA-pair kernel (2-CTA clusters sharing the B tile) where it
    applies, or the generic epilogue forced where the lean one would run. The switches are restored afterwards."""
    lib = native.load()
    lib.flpr_gemm_set_persistent(0 if name == "classic" else 1)
    lib.flpr_gemm_set_pair(1 if name == "pair" else 0)
    lib.flpr_gemm_set_generic_epilogue(1 if name == "generic-epilogue" else 0)
    try:
        yield name
    finally:
        lib.flpr_gemm_set_persistent(-1)
        lib.flpr_gemm_set_pair(-1)
        lib.flpr_gemm_set_generic_epilogue(-1)


@pytest.fixture(params=VARIANTS)
def kernel_variant(request):
    with kernel_variant_set(request.param):
        yield request.param


def gpu(fn):
    """A GPU test, run under every kernel variant."""
    return pytest.mark.gpu(pytest.mark.usefixtures("kernel_variant")(fn))


MAJORS = [(True, True), (True, False), (False, True), (False, False)]
MAJOR_IDS = ["kk", "kn", "nk", "nn"]


# ================================================================================================= CPU: the oracle
def _mutants():
    """A correct fp32 "kernel output" computed on the CPU, and deliberately wrong ones."""
    m, n, k = 96, 64, 192
    a, b, rs, cs = operands(m, n, k, seed=5)
    g = torch.Generator().manual_seed(6)
    bias = (torch.randn(n, generator=g, dtype=torch.float64) * cs * math.sqrt(k)).float()
    ref, scale = oracle(a, b, alpha=-0.75, bias_n=bias)
    A, B = a.float(), b.float()
    good = -0.75 * (A @ B.t()) + bias
    dropped = A.clone()
    dropped[:, 64:128] = 0
    wrong = {
        "dropped K block": (-0.75 * (dropped @ B.t()) + bias, False),
        "bias twice": (good + bias, False),
    }
    shifted = good.clone()
    shifted[32:64, 32:64] = good[33:65, 32:64]
    wrong["chunk shifted by a row"] = (shifted, False)
    trunc = (good.view(torch.int32) & ~0xFFFF).view(torch.float32)          # bf16 by truncation
    wrong["bf16 truncation"] = (trunc.bfloat16(), True)
    tiles = ref.abs().view(m // 32, 32, n // 32, 32).amax((1, 3))
    ti, tj = divmod(int(tiles.argmin()), n // 32)
    small = good.clone()
    small[32 * ti:32 * ti + 32, 32 * tj:32 * tj + 32] *= 1 + 1e-3
    wrong["1e-3 in the smallest tile"] = (small, False)
    return ref, scale, good, wrong, tiles


def test_oracle_accepts_correct_outputs():
    ref, scale, good, _, tiles = _mutants()
    assert float(tiles.max() / tiles.min()) > 2.0 ** 10           # the tiles differ in magnitude by orders
    assert bool(within(good, ref, scale, False).all())
    assert bool(within(good.bfloat16(), ref, scale, True).all())


@pytest.mark.parametrize("mutation", ["dropped K block", "bias twice", "chunk shifted by a row", "bf16 truncation",
                                      "1e-3 in the smallest tile"])
def test_oracle_rejects_wrong_outputs(mutation):
    ref, scale, _, wrong, _ = _mutants()
    x, bf16_out = wrong[mutation]
    assert not bool(within(x, ref, scale, bf16_out).all())


# ================================================================================================= CPU: the contract
EPILOGUES = [("bias_n",), ("bias_m",), ("bias_n", "relu"), ("residual", "relu"),
             ("bias_n", "bias_m", "residual", "relu")]
EPI_IDS = ["+".join(e) for e in EPILOGUES]


@pytest.mark.parametrize("epi", EPILOGUES, ids=EPI_IDS)
@pytest.mark.parametrize("trans_out", [False, True])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_cpu_reference_epilogue(epi, trans_out, out_dtype):
    """The CPU path of ``gemm`` is held to the same bound as the kernel."""
    gemm_case("cpu", 161, 104, 200, amaj=False, out_dtype=out_dtype, alpha=-0.75, epi=epi, trans_out=trans_out,
              out_ld=(161 if trans_out else 104) + 3)


@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_cpu_reference_col_part(out_dtype):
    """CPU statistics are those of the stored (dtype-rounded) ``alpha * A@B^T``, like the kernel's."""
    a, b, _, _ = operands(37, 40, 72, seed=3)
    part = torch.full((gops.col_part_rows(37), 2, 40), float("nan"))
    y = gops.gemm(a, b, out_dtype=out_dtype, alpha=-0.75, col_part=part)
    assert_col_part(part, y, 37)
    x = torch.randn(5, 4, 4, 64).bfloat16()
    w = (torch.randn(40, 3, 3, 64) / 24).bfloat16()
    part = torch.full((gops.col_part_rows(80), 2, 40), float("nan"))
    y = gops.conv_nhwc(x, w, out_dtype=out_dtype, alpha=-0.5, col_part=part)
    assert_col_part(part, y.reshape(-1, 40), 80)


def _refusals(dev):
    """(call, option) pairs every one of which must raise ValueError on ``dev``."""
    a, b, _, _ = operands(64, 32, 1024, seed=9)
    a, b = a.to(dev), b.to(dev)
    bias = torch.ones(32, device=dev)
    opts = {"bias_n": dict(bias_n=bias), "bias_m": dict(bias_m=torch.ones(64, device=dev)), "relu": dict(relu=True),
            "residual": dict(residual=torch.zeros(64, 32, dtype=torch.bfloat16, device=dev))}
    part = gops.col_part_buffer(64, 32, dev)
    x = torch.randn(2, 4, 4, 64, device=dev).bfloat16()
    w = torch.randn(32, 3, 3, 64, device=dev).bfloat16()
    cpart = gops.col_part_buffer(32, 32, dev)
    calls = []
    for name, kw in opts.items():
        calls.append((f"gemm split_k + {name}",
                      lambda kw=kw: gops.gemm(a, b, out_dtype=torch.float32, split_k=4, **kw)))
        calls.append((f"gemm col_part + {name}", lambda kw=kw: gops.gemm(a, b, col_part=part, **kw)))
    calls.append(("conv col_part + bias", lambda: gops.conv_nhwc(x, w, bias=bias, col_part=cpart)))
    calls.append(("conv col_part + relu", lambda: gops.conv_nhwc(x, w, relu=True, col_part=cpart)))
    calls.append(("conv col_part + residual", lambda: gops.conv_nhwc(
        x, w, residual=torch.zeros(2, 4, 4, 32, dtype=torch.bfloat16, device=dev), col_part=cpart)))
    img = torch.randn(2, 8, 8, 3, device=dev).bfloat16()
    w4 = gops.stem_weight_s2d(torch.randn(32, 3, 7, 7)).bfloat16().to(dev)
    calls.append(("stem col_part + bias", lambda: gops.stem_conv(img, w4, bias, relu=False, col_part=cpart)))
    calls.append(("stem col_part + relu", lambda: gops.stem_conv(img, w4, None, relu=True, col_part=cpart)))
    return calls


def test_cpu_refuses_split_k_and_col_part_with_epilogue():
    """Split-K would apply the epilogue once per split; ``col_part`` holds the statistics of ``alpha * A@B^T``."""
    for what, call in _refusals("cpu"):
        with pytest.raises(ValueError):
            call()
            pytest.fail(f"{what} was accepted")


def test_cpu_out_is_overwritten():
    """``out`` is overwritten on the CPU path too: ``gemm`` and the convolution weight gradient."""
    a, b, _, _ = operands(40, 24, 136, seed=4)
    out = torch.full((40, 24), 7.0)
    gops.gemm(a, b, out_dtype=torch.float32, split_k=3, out=out)
    assert torch.equal(out, gops.gemm(a, b, out_dtype=torch.float32))
    x = torch.randn(5, 4, 4, 64).bfloat16()
    dy = torch.randn(5, 4, 4, 8).bfloat16()
    slot = torch.full((8, 3, 3, 64), 7.0)
    assert gops.conv3x3_wgrad(x, dy, out=slot) is slot
    assert torch.equal(slot, gops.conv3x3_wgrad(x, dy))


def test_cpu_conv_references_within_bound():
    """The CPU convolution paths against the float64 oracle (same bound as the kernels)."""
    x, w, ref, scale = conv_problem(5, 4, 4, 64, 40, 3, 1, seed=2)
    assert_within(gops.conv_nhwc(x, w, out_dtype=torch.float32), ref, scale, False)
    dy, w, ref, scale = dgrad_problem(5, 4, 4, 64, 128, seed=2)
    assert_within(gops.conv_dgrad_nhwc(dy, w, out_dtype=torch.float32), ref, scale, False)
    x, dy, ref, scale = wgrad_problem(5, 4, 4, 64, 24, seed=2)
    assert_within(gops.conv3x3_wgrad(x, dy), ref, scale, False)


# ================================================================================================= convolution problems
def conv_problem(n, h, w, c, cout, ks, stride, seed, alpha=1.0):
    """x [n,h,w,c] with one power-of-two scale per image (several images share an M tile), w [cout,ks,ks,c] with one
    per output channel; float64 reference and scale, NHWC."""
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(n, h, w, c, generator=g, dtype=torch.float64) * _pow2(n, g, 1)[:, None, None, None]).bfloat16()
    wt = (torch.randn(cout, ks, ks, c, generator=g, dtype=torch.float64) * _pow2(cout, g)[:, None, None, None]
          ).bfloat16()
    xx, ww = x.double().permute(0, 3, 1, 2), wt.double().permute(0, 3, 1, 2)
    ref = alpha * F.conv2d(xx, ww, padding=ks // 2, stride=stride)
    scale = abs(alpha) * F.conv2d(xx.abs(), ww.abs(), padding=ks // 2, stride=stride)
    return x, wt, ref.permute(0, 2, 3, 1), scale.permute(0, 2, 3, 1)


def dgrad_problem(n, h, w, cin, cout, seed):
    g = torch.Generator().manual_seed(seed)
    dy = (torch.randn(n, h, w, cout, generator=g, dtype=torch.float64) * _pow2(n, g, 1)[:, None, None, None]).bfloat16()
    wt = (torch.randn(cout, 3, 3, cin, generator=g, dtype=torch.float64) * _pow2(cin, g)).bfloat16()
    dd, ww = dy.double().permute(0, 3, 1, 2), wt.double().permute(0, 3, 1, 2)
    ref = torch.nn.grad.conv2d_input((n, cin, h, w), ww, dd, padding=1)
    scale = torch.nn.grad.conv2d_input((n, cin, h, w), ww.abs(), dd.abs(), padding=1)
    return dy, wt, ref.permute(0, 2, 3, 1), scale.permute(0, 2, 3, 1)


def wgrad_problem(n, h, w, cin, cout, seed):
    """x scaled per input channel, dy per output channel: the rows and columns of dW [cout, 3, 3, cin]."""
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(n, h, w, cin, generator=g, dtype=torch.float64) * _pow2(cin, g)).bfloat16()
    dy = (torch.randn(n, h, w, cout, generator=g, dtype=torch.float64) * _pow2(cout, g)).bfloat16()
    xx, dd = x.double().permute(0, 3, 1, 2), dy.double().permute(0, 3, 1, 2)
    ref = torch.nn.grad.conv2d_weight(xx, (cout, cin, 3, 3), dd, padding=1)
    scale = torch.nn.grad.conv2d_weight(xx.abs(), (cout, cin, 3, 3), dd.abs(), padding=1)
    return x, dy, ref.permute(0, 2, 3, 1), scale.permute(0, 2, 3, 1)


def _wgrad_native(x, dy, out, split):
    """The weight-gradient entry point with an explicit split factor (the wrapper picks its own)."""
    lib = native.load()
    n, h, w, cin = x.shape
    cout = dy.shape[-1]
    ws = gops._split_workspace(split, cout, 9 * cin, x.device)
    rc = lib.flpr_conv_wgrad_nhwc_bf16(native.ptr(x), native.ptr(dy), native.ptr(out), n, h, w, cin, cout, 3, 3, 1, 1,
                                       int(split), 0, native.ptr(ws), native.stream(x.device))
    native.check(rc, "flpr_conv_wgrad_nhwc_bf16")


# ================================================================================================= GPU: GEMM
@gpu
@pytest.mark.parametrize("amaj,bmaj", MAJORS, ids=MAJOR_IDS)
@pytest.mark.parametrize("k", [8, 16, 40, 64, 72, 64 * 64 + 8])
def test_k_edges(k, amaj, bmaj):
    """K below one 64-wide K block, not a multiple of it, and one block past 64 blocks; every operand-major pair."""
    for out_dtype in (torch.float32, torch.bfloat16):
        gemm_case("cuda", 129, 96, k, amaj=amaj, bmaj=bmaj, out_dtype=out_dtype, alpha=-0.75, seed=k)


@gpu
@pytest.mark.parametrize("bn", [64, 128, 256])
@pytest.mark.parametrize("n", [8, 24, 40, 96, 160, 264])
@pytest.mark.parametrize("m", [1, 127, 129, 257, 3 * 128 + 1])
def test_m_n_edges(m, n, bn):
    """M around the 128-row tile (an odd tile count leaves the last CTA pair's second CTA idle), N below and around
    each tile width."""
    gemm_case("cuda", m, n, 72, bn=bn, seed=m + n)
    gemm_case("cuda", m, n, 72, amaj=False, bmaj=False, out_dtype=torch.bfloat16, bn=bn, seed=m * n)


@gpu
@pytest.mark.parametrize("amaj,bmaj", MAJORS, ids=MAJOR_IDS)
def test_strided_operands(amaj, bmaj):
    """A and B as column slices (lda, ldb > the dense width) of wider buffers, starting three rows down."""
    gemm_case("cuda", 200, 136, 200, amaj=amaj, bmaj=bmaj, pad=24, row0=3, alpha=0.5, seed=11)
    gemm_case("cuda", 129, 40, 72, amaj=amaj, bmaj=bmaj, out_dtype=torch.bfloat16, pad=8, row0=1, seed=12)


@gpu
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("extra", [8, 3], ids=["ld16B", "ld-odd"])
@pytest.mark.parametrize("m,n", [(256, 256), (161, 104)])
def test_out_view(m, n, extra, out_dtype):
    """``out`` is a view into a larger NaN-filled buffer with ldo > N; nothing outside ``[M, N]`` is written. An odd
    row stride takes the generic epilogue."""
    gemm_case("cuda", m, n, 200, out_dtype=out_dtype, out_ld=n + extra, seed=13)
    gemm_case("cuda", m, n, 200, out_dtype=out_dtype, out_ld=m + extra, trans_out=True, seed=14)
    gemm_case("cuda", m, n, 200, out_dtype=out_dtype, out_ld=n + extra, epi=("bias_n", "residual", "relu"), seed=15)


@gpu
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_out_view_misaligned(out_dtype):
    """An ``out`` (and residual) view that starts one element into its buffer: no 16-byte vector access may assume
    the row start is aligned."""
    for ld in (264, 259):
        gemm_case("cuda", 161, 256, 136, out_dtype=out_dtype, out_ld=ld, out_c0=1, seed=16)
        gemm_case("cuda", 161, 256, 136, out_dtype=out_dtype, out_ld=ld, out_c0=1, epi=("bias_n", "residual"),
                  seed=17)


@gpu
@pytest.mark.parametrize("epi", EPILOGUES, ids=EPI_IDS)
@pytest.mark.parametrize("trans_out", [False, True])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("m,n", [(256, 256), (161, 104)])
def test_epilogue_matrix(m, n, out_dtype, trans_out, epi):
    """Negative alpha != 1 with every epilogue option, fp32 / bf16 output, row-major / transposed output."""
    gemm_case("cuda", m, n, 200, out_dtype=out_dtype, alpha=-0.75, epi=epi, trans_out=trans_out, seed=m + n)


@gpu
def test_misaligned_bias_routes_to_generic_epilogue():
    """A bias that is not 16-byte aligned cannot take the lean epilogue's float4 loads; the result is still right."""
    for epi in (("bias_n",), ("bias_n", "relu"), ("bias_n", "residual", "relu")):
        gemm_case("cuda", 256, 256, 200, out_dtype=torch.bfloat16, epi=epi, bias_offset=1, seed=18)


@gpu
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("n", [40, 96, 264])
@pytest.mark.parametrize("m", [37, 161])
def test_col_part(m, n, out_dtype):
    """Fused batch-norm statistics: float64 32-row partial sums of the stored output; partial rows made only of
    padding are 0."""
    a, b, _, _ = operands(m, n, 136, seed=m + n)
    a, b = a.cuda(), b.cuda()
    ref, scale = oracle(a, b, alpha=-0.75)
    part = torch.full((gops.col_part_rows(m), 2, n), float("nan"), device="cuda")
    y = gops.gemm(a, b, out_dtype=out_dtype, alpha=-0.75, col_part=part)
    assert_within(y, ref, scale, out_dtype == torch.bfloat16)
    assert_col_part(part, y, m)


@gpu
@pytest.mark.parametrize("opt", ["bias_n", "bias_m", "relu", "residual"])
def test_split_k_refuses_epilogue(opt):
    """Split-K would run the epilogue once per split (bias added split times, ReLU of each partial, the residual read
    at each split's workspace offset): refused by the wrapper and by the library itself."""
    m, n, k = 64, 32, 1024
    a, b, _, _ = operands(m, n, k, seed=19)
    a, b = a.cuda(), b.cuda()
    kw = {"bias_n": dict(bias_n=torch.ones(n, device="cuda")), "bias_m": dict(bias_m=torch.ones(m, device="cuda")),
          "relu": dict(relu=True), "residual": dict(residual=torch.zeros(m, n, dtype=torch.bfloat16, device="cuda"))}
    with pytest.raises(ValueError):
        gops.gemm(a, b, out_dtype=torch.float32, split_k=4, **kw[opt])
    lib = native.load()
    out = torch.full((m, n), 7.0, device="cuda")
    ws = gops._split_workspace(4, m, n, a.device)
    rc = lib.flpr_gemm_bf16(native.ptr(a), native.ptr(b), native.ptr(out), m, n, k, k, k, n, 0, 0, 0, 0, 1.0,
                            native.ptr(kw[opt].get("bias_n")), native.ptr(kw[opt].get("bias_m")), int(opt == "relu"),
                            native.ptr(kw[opt].get("residual")), 4, 0, None, native.ptr(ws), native.stream(a.device))
    torch.cuda.synchronize()
    assert rc == -15
    assert bool((out == 7.0).all())


@gpu
@pytest.mark.parametrize("opt", ["bias_n", "bias_m", "relu", "residual"])
def test_col_part_refuses_epilogue(opt):
    """With bias / residual / ReLU the statistics would depend on the epilogue path (lean: after ReLU, generic staged:
    after ReLU, generic unstaged: before the residual and ReLU): refused by the wrapper and by the library."""
    m, n, k = 161, 264, 136
    a, b, _, _ = operands(m, n, k, seed=20)
    a, b = a.cuda(), b.cuda()
    kw = {"bias_n": dict(bias_n=torch.ones(n, device="cuda")), "bias_m": dict(bias_m=torch.ones(m, device="cuda")),
          "relu": dict(relu=True), "residual": dict(residual=torch.zeros(m, n, dtype=torch.bfloat16, device="cuda"))}
    part = gops.col_part_buffer(m, n, "cuda")
    with pytest.raises(ValueError):
        gops.gemm(a, b, col_part=part, **kw[opt])
    lib = native.load()
    out = torch.empty(m, n, dtype=torch.bfloat16, device="cuda")
    rc = lib.flpr_gemm_bf16(native.ptr(a), native.ptr(b), native.ptr(out), m, n, k, k, k, n, 0, 0, 1, 0, 1.0,
                            native.ptr(kw[opt].get("bias_n")), native.ptr(kw[opt].get("bias_m")), int(opt == "relu"),
                            native.ptr(kw[opt].get("residual")), 1, 0, native.ptr(part), None,
                            native.stream(a.device))
    assert rc == -16
    x = torch.randn(2, 4, 4, 64, device="cuda").bfloat16()
    w = torch.randn(32, 3, 3, 64, device="cuda").bfloat16()
    cpart = gops.col_part_buffer(32, 32, "cuda")
    if opt == "bias_n":
        with pytest.raises(ValueError):
            gops.conv_nhwc(x, w, bias=torch.ones(32, device="cuda"), col_part=cpart)
    elif opt == "relu":
        with pytest.raises(ValueError):
            gops.stem_conv(torch.randn(2, 8, 8, 3, device="cuda").bfloat16(),
                           gops.stem_weight_s2d(torch.randn(32, 3, 7, 7)).bfloat16().cuda(), None, relu=True,
                           col_part=cpart)


@gpu
@pytest.mark.parametrize("trans_out", [False, True])
@pytest.mark.parametrize("split", [2, 3, 7, 16, 21])
def test_split_k(split, trans_out):
    """K = 1000 (16 K blocks, not a multiple of 64 * split; 7 gives 6 splits of 3, 21 is clamped to 16), alpha != 1,
    ``out`` a strided view pre-filled with garbage: the splits' sum overwrites it."""
    gemm_case("cuda", 200, 72, 1000, alpha=-0.75, split_k=split, trans_out=trans_out,
              out_ld=(200 if trans_out else 72) + 5, prefill=True, seed=split)
    gemm_case("cuda", 129, 64, 1000, amaj=False, bmaj=False, split_k=split, out_ld=64, prefill=True, seed=split + 1)


# ================================================================================================= GPU: convolutions
@gpu
@pytest.mark.parametrize("epi", ["plain", "bias+relu", "bias+residual+relu"])
@pytest.mark.parametrize("n,h,w,c,cout,ks,stride", [
    (5, 4, 4, 64, 96, 3, 1),       # 8 images per M tile, 5 present
    (3, 1, 1, 128, 64, 3, 1),      # 1x1 maps under a 3x3 kernel: 128 images per tile
    (7, 2, 2, 64, 40, 3, 1),       # 2x2 maps, Cout not a multiple of 32
    (5, 4, 4, 64, 64, 1, 1),
    (3, 7, 8, 64, 64, 3, 2),       # stride 2 on an odd H
    (2, 15, 15, 64, 128, 3, 2),
    (3, 7, 8, 128, 64, 1, 2),
], ids=["pack5of8", "1x1map", "2x2map", "k1", "s2-oddH", "s2-15x15", "k1s2-oddH"])
def test_conv_nhwc(n, h, w, c, cout, ks, stride, epi):
    x, wt, ref, scale = conv_problem(n, h, w, c, cout, ks, stride, seed=n * h + cout, alpha=-0.5)
    bias = res = None
    g = torch.Generator().manual_seed(21)
    if "bias" in epi:
        bias = torch.randn(cout, generator=g) * scale.mean((0, 1, 2)).float()
        ref, scale = ref + bias.double(), scale + bias.double().abs()
    if "residual" in epi:
        res = (torch.randn(ref.shape, generator=g, dtype=torch.float64) * scale).bfloat16()
        ref, scale = ref + res.double(), scale + res.double().abs()
    if "relu" in epi:
        ref = ref.clamp_min(0)
    for out_dtype in (torch.float32, torch.bfloat16):
        y = gops.conv_nhwc(x.cuda(), wt.cuda(), padding=ks // 2, stride=stride, out_dtype=out_dtype, alpha=-0.5,
                           bias=None if bias is None else bias.cuda(), relu="relu" in epi,
                           residual=None if res is None else res.cuda())
        assert_within(y.cpu(), ref, scale, out_dtype == torch.bfloat16)


@gpu
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("n,h,w,c,cout", [(5, 4, 4, 64, 96), (3, 7, 8, 64, 40), (9, 2, 2, 64, 264)])
def test_conv_col_part(n, h, w, c, cout, out_dtype):
    """Convolution statistics with a partly filled last M tile (and a stride-2 / odd-H case)."""
    stride = 2 if h == 7 else 1
    x, wt, ref, scale = conv_problem(n, h, w, c, cout, 3, stride, seed=cout, alpha=-0.5)
    m = ref.shape[0] * ref.shape[1] * ref.shape[2]
    part = torch.full((gops.col_part_rows(m), 2, cout), float("nan"), device="cuda")
    y = gops.conv_nhwc(x.cuda(), wt.cuda(), stride=stride, out_dtype=out_dtype, alpha=-0.5, col_part=part)
    assert_within(y.cpu(), ref, scale, out_dtype == torch.bfloat16)
    assert_col_part(part.cpu(), y.reshape(-1, cout).cpu(), m)


@gpu
@pytest.mark.parametrize("bn", [64, 256])
@pytest.mark.parametrize("n,h,w,cin,cout", [(5, 4, 4, 64, 64), (5, 4, 4, 256, 128), (7, 2, 2, 128, 64),
                                            (3, 8, 16, 64, 128)])
def test_conv_dgrad(n, h, w, cin, cout, bn):
    """Data gradient with several images packed per M tile, N below and equal to the 256-wide tile."""
    dy, wt, ref, scale = dgrad_problem(n, h, w, cin, cout, seed=cin + n)
    for out_dtype in (torch.float32, torch.bfloat16):
        y = gops.conv_dgrad_nhwc(dy.cuda(), wt.cuda(), out_dtype=out_dtype, bn=bn)
        assert_within(y.cpu(), ref, scale, out_dtype == torch.bfloat16)


@gpu
@pytest.mark.parametrize("n,h,w,cin,cout", [(5, 4, 4, 64, 8), (5, 4, 4, 64, 24), (9, 2, 2, 64, 24),
                                            (49, 4, 4, 64, 8), (64, 8, 8, 128, 64)])
def test_conv3x3_wgrad_overwrites(n, h, w, cin, cout):
    """Weight gradient through the wrapper (its own split factor: 1, or 3 of 13 K blocks for 49 4x4 images, or 13 of
    64 for the long K) into a slot holding garbage: the slot is overwritten. NIMG*H*W need not be a multiple of
    64."""
    x, dy, ref, scale = wgrad_problem(n, h, w, cin, cout, seed=n + cout)
    slot = torch.full((cout, 3, 3, cin), 1e3, device="cuda")
    assert gops.conv3x3_wgrad(x.cuda(), dy.cuda(), out=slot) is slot
    assert_within(slot.cpu(), ref, scale, False)
    assert_within(gops.conv3x3_wgrad(x.cuda(), dy.cuda()).cpu(), ref, scale, False)


@gpu
@pytest.mark.parametrize("cout", [8, 24])
@pytest.mark.parametrize("split", [2, 3, 7, 13, 20])
def test_conv3x3_wgrad_split(split, cout):
    """Explicit split factors over 13 K blocks (784 pixels: the last block is partial): 2, 3 and 7 do not divide 13,
    20 is clamped. ``out`` holds garbage and is overwritten."""
    x, dy, ref, scale = wgrad_problem(49, 4, 4, 64, cout, seed=split)
    out = torch.full((cout, 3, 3, 64), -5.0, device="cuda")
    _wgrad_native(x.cuda().contiguous(), dy.cuda().contiguous(), out, split)
    assert_within(out.cpu(), ref, scale, False)


# ================================================================================================= GPU: variants agree
def _variant_outputs(case):
    """The outputs of one fixed-``bn`` problem under the current kernel variant."""
    if case == "gemm":
        a, b, _, _ = operands(257, 200, 520, seed=30)
        a, b = a.cuda(), b.cuda()
        return [gops.gemm(a, b, out_dtype=torch.float32, alpha=-0.75, bn=128),
                gops.gemm(a, b, out_dtype=torch.bfloat16, alpha=-0.75, bn=128),
                gops.gemm(a, b, out_dtype=torch.float32, trans_out=True, bn=128)]
    if case == "bias-relu":
        a, b, _, cs = operands(257, 256, 520, seed=31)
        bias = (torch.randn(256, generator=torch.Generator().manual_seed(3), dtype=torch.float64) * cs * 20).float()
        return [gops.gemm(a.cuda(), b.cuda(), bias_n=bias.cuda(), relu=True, bn=128)]
    if case == "col-part":
        a, b, _, _ = operands(257, 256, 520, seed=32)
        part = gops.col_part_buffer(257, 256, "cuda")
        return [gops.gemm(a.cuda(), b.cuda(), col_part=part, bn=128), part]
    if case == "split-k":
        a, b, _, _ = operands(257, 128, 2000, seed=33)
        return [gops.gemm(a.cuda(), b.cuda(), out_dtype=torch.float32, split_k=5, bn=128)]
    if case == "conv":
        x, wt, _, _ = conv_problem(5, 4, 4, 64, 256, 3, 1, seed=34)
        part = gops.col_part_buffer(80, 256, "cuda")
        return [gops.conv_nhwc(x.cuda(), wt.cuda(), bn=128, col_part=part), part,
                gops.conv_dgrad_nhwc(x.cuda(), wt.cuda().permute(3, 1, 2, 0).contiguous(), bn=128)]
    x, dy, _, _ = wgrad_problem(49, 4, 4, 64, 24, seed=35)
    return [gops.conv3x3_wgrad(x.cuda(), dy.cuda())]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["gemm", "bias-relu", "col-part", "split-k", "conv", "wgrad"])
def test_variants_agree_bitwise(case):
    """With the tile width pinned, every kernel variant runs the same K order per output tile and the same epilogue
    arithmetic: the results agree bit for bit."""
    outs = {}
    for v in VARIANTS:
        with kernel_variant_set(v):
            outs[v] = [t.clone() for t in _variant_outputs(case)]
    for v in VARIANTS[1:]:
        for i, (t, t0) in enumerate(zip(outs[v], outs[VARIANTS[0]])):
            assert torch.equal(_bits(t), _bits(t0)), f"{case} output {i}: {v} differs from {VARIANTS[0]}"

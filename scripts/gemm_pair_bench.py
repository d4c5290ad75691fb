"""CTA-pair kernel (2-CTA clusters, B tile multicast) vs the single-CTA persistent kernel on the head-step shapes."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch
from flpr_b200.ops import native
from flpr_b200.ops.gemm import gemm, conv_nhwc, conv_dgrad_nhwc, conv3x3_wgrad
from gemm_bench import timeit
lib = native.load()
torch.manual_seed(0)
for (m, n, k) in [(8192, 2048, 512), (8192, 512, 2048), (8192, 2048, 2048), (32768, 2048, 512)]:
    a = torch.randn(m, k, device="cuda").bfloat16(); b = (torch.randn(n, k, device="cuda") / k ** 0.5).bfloat16()
    ref = a.float() @ b.float().t()
    for pair in (0, 1):
        lib.flpr_gemm_set_pair(pair)
        out = gemm(a, b, bn=256)
        err = (out.float() - ref).abs().max().item()
        t = timeit(lambda: gemm(a, b, bn=256))
        print(f"{(m, n, k)} pair={pair}: {t:7.1f} us ({2.0 * m * n * k / t / 1e6:7.1f} TF)  max err {err:.3f}")
x = torch.randn(64, 16, 8, 512, device="cuda").bfloat16()
w = (torch.randn(512, 3, 3, 512, device="cuda") / 60).bfloat16()
dy = torch.randn(64, 16, 8, 512, device="cuda").bfloat16()
fl = 2.0 * 8192 * 512 * 4608
for pair in (0, 1):
    lib.flpr_gemm_set_pair(pair)
    y = conv_nhwc(x, w, padding=1, bn=256)
    t = timeit(lambda: conv_nhwc(x, w, padding=1, bn=256))
    t2 = timeit(lambda: conv_dgrad_nhwc(dy, w, padding=1, bn=256))
    print(f"conv3x3 fwd pair={pair}: {t:7.1f} us ({fl / t / 1e6:7.1f} TF)   dgrad {t2:7.1f} us   |y| {y.float().abs().mean().item():.4f}")
lib.flpr_gemm_set_pair(-1)

"""Isolated timing of the wgmma GEMM on the head-step shapes: persistent vs classic kernel, tile widths, fused
statistics on/off, next to torch.matmul (cuBLAS) on the same shapes. CUDA events, L2 flushed between iterations."""
import os, sys, math
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from flpr_b200.ops import native
from flpr_b200.ops.gemm import gemm, conv_nhwc, conv3x3_wgrad, conv_dgrad_nhwc, col_part_buffer


def timeit(fn, iters=20):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for _ in range(3):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def main():
    lib = native.load()
    torch.manual_seed(0)
    shapes = [(8192, 2048, 512), (8192, 512, 1024), (8192, 512, 2048), (8192, 2048, 1024), (32768, 2048, 512),
              (64, 8000, 2048)]
    print(f"{'shape':>22s} {'cfg':>28s} {'us':>8s} {'TFLOP/s':>8s}")
    for m, n, k in shapes:
        a = torch.randn(m, k, device="cuda").bfloat16()
        b = torch.randn(n, k, device="cuda").bfloat16()
        fl = 2.0 * m * n * k
        t = timeit(lambda: torch.matmul(a, b.t()))
        print(f"{str((m, n, k)):>22s} {'cuBLAS (torch.matmul)':>28s} {t:8.1f} {fl / t / 1e6:8.1f}")
        for persist in (1, 0):
            lib.flpr_gemm_set_persistent(persist)
            for bn in (128, 256):
                for stats in (0, 1):
                    part = col_part_buffer(m, n, "cuda") if stats else None
                    t = timeit(lambda: gemm(a, b, bn=bn, col_part=part))
                    print(f"{str((m, n, k)):>22s} {f'persist={persist} bn={bn} stats={stats}':>28s} {t:8.1f} {fl / t / 1e6:8.1f}")
        lib.flpr_gemm_set_persistent(1)
    # 3x3 conv forward / dgrad / wgrad on the layer4 shape
    x = torch.randn(64, 16, 8, 512, device="cuda").bfloat16()
    w = (torch.randn(512, 3, 3, 512, device="cuda") / 60).bfloat16()
    dy = torch.randn(64, 16, 8, 512, device="cuda").bfloat16()
    fl = 2.0 * 8192 * 512 * 4608
    for persist in (1, 0):
        lib.flpr_gemm_set_persistent(persist)
        for bn in (128, 256):
            t = timeit(lambda: conv_nhwc(x, w, padding=1, bn=bn))
            print(f"{'conv3x3 fwd':>22s} {f'persist={persist} bn={bn}':>28s} {t:8.1f} {fl / t / 1e6:8.1f}")
            t = timeit(lambda: conv_dgrad_nhwc(dy, w, padding=1, bn=bn))
            print(f"{'conv3x3 dgrad':>22s} {f'persist={persist} bn={bn}':>28s} {t:8.1f} {fl / t / 1e6:8.1f}")
        out = torch.zeros(512, 3, 3, 512, device="cuda")
        t = timeit(lambda: conv3x3_wgrad(x, dy, out=out))
        print(f"{'conv3x3 wgrad':>22s} {f'persist={persist}':>28s} {t:8.1f} {fl / t / 1e6:8.1f}")
    lib.flpr_gemm_set_persistent(1)
    xt = x.permute(0, 3, 1, 2)
    wt = w.permute(0, 3, 1, 2)
    t = timeit(lambda: torch.nn.functional.conv2d(xt, wt, padding=1))
    print(f"{'conv3x3 fwd':>22s} {'cuDNN (channels_last)':>28s} {t:8.1f} {fl / t / 1e6:8.1f}")


if __name__ == "__main__":
    main()

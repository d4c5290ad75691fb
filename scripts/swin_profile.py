"""Where does a Swin-T forward (frozen trunk, eval) / head step spend its device and host time? (torch.profiler)"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import ProfilerActivity, profile
from flpr_b200.runtime.builder import parser_model

dev = torch.device("cuda:0")
cfg = {"name": "swin_transformer_tiny", "num_classes": 8000, "neck": "bnneck", "atten_default": 0.9, "lambda_l1": 1e-3,
       "lambda_k": 64, "fine_tuning": ["base.layers.3", "classifier"]}
model = parser_model("fedstil", cfg, dev, {"compute_dtype": "bf16"})
x = torch.randn(64, 3, 256, 128, device=dev).to(torch.bfloat16)
model.eval()


def trunk():
    with torch.no_grad(), model.autocast():
        return model.forward_trunk(x)


from flpr_b200.ops import native
for tc in (0, 1):
    native.load().flpr_window_attn_set_tc(tc)
    for _ in range(3):
        trunk()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(5):
        trunk()
    torch.cuda.synchronize()
    print(f"trunk fwd, batch 64, wgmma attention {'on' if tc else 'off'}: {(time.perf_counter() - t0) / 5 * 1e3:.2f} ms wall")
with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
    trunk()
    torch.cuda.synchronize()
print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=22, max_name_column_width=70))

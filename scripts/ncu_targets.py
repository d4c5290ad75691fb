"""A small workload that launches every kernel family once or twice (for `ncu -k regex:<family>`):

    ncu --set full --clock-control none --import-source on -k regex:<pattern> -c 4 -o gpurun_out/prof_<x> \
        python scripts/ncu_targets.py <what>

what: head (FedSTIL ResNet-50 head step: wgmma GEMM / conv fwd, dgrad, wgrad, BN, CE, fused Adam + trained anchor),
      trunk (native train-mode trunk: stem, strided convs, batch-stat BN), swin (wgmma window attention + TcLinear),
      comm (fed_mix / fed_reduce_bcast / gather on one GPU), misc (triplet mining, herding, augmentation, rank_eval).
"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from flpr_b200.runtime.builder import parser_criterion, parser_model
from flpr_b200.runtime.arena import ArenaOptimizer

what = sys.argv[1] if len(sys.argv) > 1 else "head"
dev = torch.device("cuda:0")
torch.manual_seed(0)
R50 = {"name": "resnet50", "num_classes": 8000, "last_stride": 1, "neck": "bnneck", "atten_default": 0.9,
       "lambda_l1": 1e-3, "lambda_k": 64, "fine_tuning": ["base.layer4", "classifier"]}

if what == "head":
    model = parser_model("fedstil", R50, dev, {"compute_dtype": "bf16"})
    crit = parser_criterion({"name": "cross_entropy", "num_classes": 8000, "epsilon": 0.1})[0]
    opt = ArenaOptimizer("adam", model.arena, lr=1e-3, weight_decay=1e-5)
    model.train_l1_anchor = True
    model.install(opt)
    proto = (torch.randn(64, 1024, 16, 8, device=dev) * 0.5).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 8000, (64,), device=dev)
    model.train()
    for _ in range(int(os.environ.get('NSTEPS', '3'))):
        opt.zero_grad()
        with model.autocast():
            score, feat = model.forward_head(proto)
        crit(score=score, feature=feat, target=y).backward()
        opt.step()
elif what == "trunk":
    model = parser_model("fedavg", {k: v for k, v in R50.items() if k not in ("atten_default", "lambda_l1", "lambda_k")},
                         dev, {"compute_dtype": "bf16"})
    x = torch.randn(64, 3, 256, 128, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    model.train()
    for _ in range(2):
        with torch.no_grad():
            model.net.forward_trunk(x)
elif what == "swin":
    cfg = {"name": "swin_transformer_tiny", "num_classes": 8000, "neck": "bnneck", "atten_default": 0.9,
           "lambda_l1": 1e-3, "lambda_k": 64, "fine_tuning": ["base.layers.3", "classifier"]}
    model = parser_model("fedstil", cfg, dev, {"compute_dtype": "bf16"})
    x = torch.randn(64, 3, 256, 128, device=dev).to(torch.bfloat16)
    model.eval()
    for _ in range(2):
        with torch.no_grad(), model.autocast():
            model.forward_trunk(x)
elif what == "comm":
    from flpr_b200.parallel.comm import FedComm
    n = 31_326_208
    comm = FedComm(dev, 8, arena_bytes=n * 4 * 11 + (16 << 20))
    comm.alloc_client_buffer("theta_up", n)
    comm.alloc_rank_buffer("glob", n)
    for c in range(8):
        comm.client_view("theta_up", c).normal_()
    dst = [torch.empty(n, device=dev) for _ in range(2)]
    dstb = [torch.empty(n, device=dev, dtype=torch.bfloat16) for _ in range(2)]
    rows = torch.softmax(torch.randn(2, 8, device=dev), 1)
    for _ in range(2):
        comm.reduce_bcast("theta_up", "glob", list(range(8)), weights=[0.125] * 8)
        comm.mix("theta_up", list(range(8)), rows, [0, 1], dst, dst, dstb)
    out = torch.empty(n, 8, device=dev)
    comm.gather_strided("theta_up", list(range(8)), out)
    torch.cuda.synchronize()
    comm.close()
else:
    from flpr_b200.criterions import TripletLoss
    from flpr_b200.methods.fedstil import herding_select_batched
    from flpr_b200.ops.rank import rank_metrics, similarity
    from flpr_b200.data.augmentation import DeviceAugment
    x = torch.randn(64, 2048, device=dev, requires_grad=True)
    lab = torch.arange(16, device=dev).repeat_interleave(4)
    for hard in (True, False):
        TripletLoss(margin=0.3, hard_mining=hard)(feature=x, target=lab).backward()
    feats = torch.randn(1024, 2048, device=dev)
    idx = torch.arange(1024, device=dev).view(64, 16)
    herding_select_batched(feats, idx, torch.full((64,), 16, device=dev), 8)
    q, g = torch.nn.functional.normalize(torch.randn(512, 2048, device=dev)), torch.nn.functional.normalize(torch.randn(4096, 2048, device=dev))
    rank_metrics(similarity(q, g), torch.randint(0, 100, (512,), device=dev), torch.randint(0, 100, (4096,), device=dev))
    try:
        aug = DeviceAugment("default", dtype=torch.bfloat16)
        aug(torch.randint(0, 256, (256, 256, 128, 3), dtype=torch.uint8, device=dev), None)
    except Exception as ex:
        print("augment skipped:", ex)
torch.cuda.synchronize()
print("ncu target", what, "done")

"""Fused NetVLAD kernel check + timing (GPU): tensor-core path (nhwc) against the fp32 CUDA-core path (nchw) for a
few shapes, then the device time of the kernels at B=32, S=1200 (cold L2 between reps: 256 MB scratch write)."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from openibl_b200 import synth
from openibl_b200.engine import Engine

eng = Engine.get(0)
for sharp in (False, True):
    p = synth.make_netvlad_params(seed=8, sharp=sharp)
    w, c = p["conv_weight"].cuda(), p["centroids"].cuda()
    for (B, H, W) in ((1, 30, 40), (2, 7, 9), (3, 16, 8), (5, 30, 40), (32, 30, 40), (40, 12, 20)):
        torch.manual_seed(B * 100 + H)
        feat = torch.randn(B, H, W, 512, device="cuda")
        t0 = time.time()
        raw, nrm = eng.netvlad_forward(feat, w, c, nhwc=True, want_raw=True, want_norm=True)
        torch.cuda.synchronize()
        raw2, nrm2 = eng.netvlad_forward(feat.permute(0, 3, 1, 2).contiguous(), w, c, nhwc=False, want_raw=True, want_norm=True)
        torch.cuda.synchronize()
        e1 = float((raw - raw2).norm() / raw2.norm()); e2 = float((nrm - nrm2).norm() / nrm2.norm())
        print(f"sharp={sharp} B={B} S={H*W}: raw rel {e1:.2e}  norm rel {e2:.2e}  {'OK' if e1 < 1e-4 and e2 < 1e-4 else 'MISMATCH'}", flush=True)

p = synth.make_netvlad_params(seed=8, sharp=True)
w, c = p["conv_weight"].cuda(), p["centroids"].cuda()
feat = torch.randn(32, 30, 40, 512, device="cuda")
scratch = torch.empty(64 * 1024 * 1024, device="cuda")
for _ in range(3):
    eng.netvlad_forward(feat, w, c, nhwc=True, want_raw=False, want_norm=True)
ts = []
for _ in range(10):
    scratch.zero_()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    eng.netvlad_forward(feat, w, c, nhwc=True, want_raw=False, want_norm=True)
    b.record()
    torch.cuda.synchronize()
    ts.append(a.elapsed_time(b) * 1e3)
print("whole call (planes + sqnorm + fused + 2 finalize), us:", [round(t, 1) for t in ts])

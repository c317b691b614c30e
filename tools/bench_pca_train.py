#!/usr/bin/env python
"""Times the PCA layer's training kernels at the hub model's shape (P = 4096, D = 32768) and one full fine-tuning
step of the hub model, and prints one JSON line.

  forward  y = v W^T + b         ibl_pca_forward_train   bytes: the W planes (2 x P x D bf16) + v + y
  dgrad    gv = gy W             ibl_pca_backward(gv)    bytes: the W planes + gy + gv
  wgrad    gW = gy^T v, gb       ibl_pca_backward(gW,gb) bytes: the fp32 gW store (P x D x 4) + v + gy
  step     EmbedNetPCA (conv5, NetVLAD and PCA trainable) forward + triplet loss + backward + SGD step at 480 x 640

Achieved GB/s = those bytes over the CUDA-event time of the call, against the H100 SXM's 3.35 TB/s HBM3 data-sheet
peak.  The card's name and power limit are read in the same run.

    python tools/bench_pca_train.py [--iters 20] [--batches 12,48,88]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
HBM_PEAK_GBS = 3350.0


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--batches", default="12,48,88")
    ap.add_argument("--step-images", type=int, default=12)
    args = ap.parse_args()
    from openibl_b200.engine import Engine
    from openibl_b200 import synth
    assert torch.cuda.is_available(), "bench_pca_train needs a GPU"
    eng = Engine.get(0)
    P, D = 4096, 32768
    g = torch.Generator(device="cuda").manual_seed(0)
    W = (torch.rand(P, D, device="cuda", generator=g) * 2 - 1) / D ** 0.5
    b = torch.zeros(P, device="cuda")
    eng.set_pca(W, b, force=True)
    planes = 2 * P * D * 2
    rows = []
    for N in [int(n) for n in args.batches.split(",")]:
        v = torch.nn.functional.normalize(torch.randn(N, D, device="cuda", generator=g), dim=1)
        gy = torch.randn(N, P, device="cuda", generator=g)
        t_f = timed(lambda: eng.pca_forward_train(v, W, b), args.iters)
        t_d = timed(lambda: eng.pca_backward(v, W, gy, need_gw=False, need_gb=False), args.iters)
        t_w = timed(lambda: eng.pca_backward(v, W, gy, need_gv=False), args.iters)
        by_f = planes + N * D * 4 + N * P * 4
        by_d = planes + N * P * 4 + N * D * 4
        by_w = P * D * 4 + N * D * 4 + N * P * 4
        rows.append({"N": N, **{f"{k}_ms": round(t, 4) for k, t in (("forward", t_f), ("dgrad", t_d), ("wgrad", t_w))},
                     **{f"{k}_GBps": round(by / t / 1e6, 1) for k, by, t in
                        (("forward", by_f, t_f), ("dgrad", by_d, t_d), ("wgrad", by_w, t_w))},
                     **{f"{k}_of_hbm_peak": round(by / t / 1e6 / HBM_PEAK_GBS, 3) for k, by, t in
                        (("forward", by_f, t_f), ("dgrad", by_d, t_d), ("wgrad", by_w, t_w))}})
    del W, v, gy
    # one fine-tuning step of the hub model at 480 x 640
    from ibl import models
    base = models.create("vgg16", pretrained=False)
    model = models.create("embednetpca", base, models.create("netvlad", dim=512), dim=4096)
    model.load_state_dict(synth.make_state_dict(seed=1, sharp=True, with_pca=True, bias_scale=0.02))
    for layer in list(model.base_model.base.children())[:24]:
        for p in layer.parameters():
            p.requires_grad = False
    model.cuda().train()
    opt = torch.optim.SGD([p for p in model.parameters() if p.requires_grad], lr=1e-3, momentum=0.9)
    x = synth.make_smooth_images(2, args.step_images, 480, 640).cuda()

    def step():
        out = model(x).view(1, args.step_images, -1)
        neg = out[:, 2:].reshape(-1, out.shape[-1])
        anc = out[:, 0].expand_as(out[0, 2:])
        pos = out[:, 1].expand_as(out[0, 2:])
        loss = torch.nn.functional.triplet_margin_loss(anc, pos, neg, margin=0.1 ** 0.5)
        opt.zero_grad()
        loss.backward()
        opt.step()

    t_step = timed(step, max(3, args.iters // 4))
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    print("BENCH_PCA_TRAIN " + json.dumps({"gpu": smi[0] if smi else torch.cuda.get_device_name(0), "P": P, "D": D,
                                           "pca": rows, "step_images": args.step_images, "step_480x640_ms":
                                           round(t_step, 2)}), flush=True)


if __name__ == "__main__":
    main()

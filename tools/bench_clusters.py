#!/usr/bin/env python
"""Cost of NetVLAD layers with fewer than 64 clusters.

For K in --clusters: extraction images/s (batch 32, 480x640, PCA K*512 -> 4096, device-resident inputs) and the
raw-descriptor ranking (top-10 of --queries queries against --db rows of width K*512).  The tensor-core NetVLAD
kernel pads K < 64 to 64 clusters, so extraction does K = 64 NetVLAD work whatever K is; the PCA layer and the
ranking see the narrower K*512 descriptor.  Prints one JSON line with the card name and its power limit.

    python tools/bench_clusters.py --steps 20
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from openibl_b200 import synth  # noqa: E402
from openibl_b200.engine import CONV_TC_BF16X3, Engine  # noqa: E402

BATCH, H, W, PCA_DIM = 32, 480, 640, 4096


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30)
        return float(out.stdout.strip().splitlines()[0])
    except Exception:
        return None


def timed(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clusters", default="16,32,64")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--queries", type=int, default=1000)
    ap.add_argument("--db", type=int, default=20000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_clusters.py needs an H100: the engine has no CPU fallback")
    dev = torch.device("cuda", 0)
    eng = Engine.get(0)
    eng.conv_mode = CONV_TC_BF16X3
    eng.set_gemm_mode(1)
    xs = [synth.make_images(seed=100 + i, batch=BATCH).to(dev) for i in range(2)]
    gen = torch.Generator(device=dev).manual_seed(7)
    rows = []
    for K in [int(k) for k in args.clusters.split(",")]:
        sd = {k: v.to(dev) for k, v in synth.make_state_dict(seed=0, with_pca=True, pca_dim=PCA_DIM,
                                                             num_clusters=K).items()}
        slots = synth.VGG16_CONV_SLOTS
        eng.set_vgg16([sd[f"base_model.base.{s}.weight"] for s in slots],
                      [sd[f"base_model.base.{s}.bias"] for s in slots], force=True)
        eng.set_netvlad(sd["net_vlad.conv.weight"], sd["net_vlad.centroids"])
        eng.set_pca(sd["pca_layer.weight"], sd["pca_layer.bias"], force=True)
        for i in range(args.warmup):
            eng.extract(xs[i % 2], pca=True)
        torch.cuda.synchronize()
        ms = timed(lambda i: eng.extract(xs[i % 2], pca=True), args.steps)
        D = K * 512
        db = torch.nn.functional.normalize(torch.randn(args.db, D, device=dev, generator=gen), dim=1)
        q = torch.nn.functional.normalize(db[: args.queries] + 0.2 * torch.randn(args.queries, D, device=dev,
                                                                                  generator=gen), dim=1)
        eng.l2dist_topk(q, db, 10)
        torch.cuda.synchronize()
        rank_ms = timed(lambda i: eng.l2dist_topk(q, db, 10), max(3, args.steps // 4))
        rows.append({"clusters": K, "raw_dim": D, "extract_ms_per_batch": ms,
                     "extract_images_per_s": BATCH * 1000.0 / ms,
                     "rank_raw_ms": rank_ms, "rank_shape": [args.queries, args.db, D]})
        del sd, db, q
        torch.cuda.empty_cache()
    print(json.dumps({"metric": "netvlad_clusters_cost", "device": torch.cuda.get_device_name(0),
                      "power_limit_w": power_limit_w(), "batch": BATCH, "image": [H, W], "pca_dim": PCA_DIM,
                      "steps": args.steps, "rows": rows}))


if __name__ == "__main__":
    main()

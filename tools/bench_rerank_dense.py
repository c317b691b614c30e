#!/usr/bin/env python
"""Measure the SFRS sampler refresh's re-ranking call, re_ranking(host q-g, q-q, g-g, k1=20, k2=1, lambda=0.1)
(examples/netvlad_img_sfrs.py:84), at the Pitts30k-train shape.

    python tools/bench_rerank_dense.py                              # 7,416 queries x 10,000 gallery, d = 4096
    python tools/bench_rerank_dense.py --host-q 1854 --host-db 2500  # host torch leg on a subset

Synthetic make_gallery descriptors; the distances come from Engine.l2dist_dense and are moved to the host, as the
driver's pairwise_distance leaves them.  Prints one JSON line:
  host_route_ms      re_ranking on numpy arrays (copies to the device, Engine.rerank_dense, copy back)
  device_ms          Engine.rerank_dense on device inputs, CUDA events
  torch_gpu_ms       the dense torch restatement on the same GPU (re_ranking(..., device="cuda"))
  torch_host_ms      the dense torch restatement on the host cores, on the first --host-q queries and --host-db gallery
                     rows (the full shape takes many minutes there); host_subset gives that shape
  peak_above_io_bytes  device memory the device path holds above its inputs and output: torch's peak plus the
                     engine's re-ranking workspace
  max_abs_diff_vs_torch  device path against the torch restatement on the GPU, full shape
  card, power_limit, sm_clock  read in the same call
Refuses to run without a GPU."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from openibl_b200 import synth  # noqa: E402
from openibl_b200.engine import Engine  # noqa: E402
from openibl_b200.utils.rerank import re_ranking  # noqa: E402


def card():
    name = torch.cuda.get_device_name()
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        parts = [p.strip() for p in r.stdout.strip().split(",")]
        power, clock = (parts + [None, None])[:2]
    except Exception:
        power = clock = None
    return name, power, clock


def timed(fn, reps):
    """median wall time of fn() in ms; fn ends in a device synchronise"""
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-q", type=int, default=7416)
    ap.add_argument("--n-db", type=int, default=10000)
    ap.add_argument("--dim", type=int, default=4096)
    ap.add_argument("--k1", type=int, default=20)
    ap.add_argument("--k2", type=int, default=1)
    ap.add_argument("--lambda-value", type=float, default=0.1)
    ap.add_argument("--host-q", type=int, default=1854)
    ap.add_argument("--host-db", type=int, default=2500)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--skip-host-torch", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_rerank_dense.py measures the H100 path and needs a CUDA device")
    eng = Engine.get(0)
    k1, k2, lam = args.k1, args.k2, args.lambda_value
    q, db, _ = synth.make_gallery(n_db=args.n_db, n_q=args.n_q, dim=args.dim)
    q, db = q.cuda(), db.cuda()
    qg_d, qq_d, gg_d = eng.l2dist_dense(q, db), eng.l2dist_dense(q, q), eng.l2dist_dense(db, db)
    del q, db
    qg, qq, gg = (a.cpu().numpy() for a in (qg_d, qq_d, gg_d))
    out = dict(m=args.n_q, n=args.n_db, dim=args.dim, k1=k1, k2=k2, lambda_value=lam)

    re_ranking(qg, qq, gg, k1=k1, k2=k2, lambda_value=lam)                  # warm-up (module load, workspaces)
    out["host_route_ms"] = timed(lambda: re_ranking(qg, qq, gg, k1=k1, k2=k2, lambda_value=lam), args.reps)

    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    final = eng.rerank_dense(qg_d, qq_d, gg_d, k1, k2, lam)
    torch.cuda.synchronize()
    out["peak_above_io_bytes"] = (torch.cuda.max_memory_allocated() - base - final.numel() * 4
                                  + eng.rerank_workspace_bytes())
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ts = []
    for _ in range(args.reps):
        ev[0].record()
        eng.rerank_dense(qg_d, qq_d, gg_d, k1, k2, lam)
        ev[1].record()
        torch.cuda.synchronize()
        ts.append(ev[0].elapsed_time(ev[1]))
    out["device_ms"] = sorted(ts)[len(ts) // 2]

    want = re_ranking(qg_d, qq_d, gg_d, k1=k1, k2=k2, lambda_value=lam, device="cuda")
    out["max_abs_diff_vs_torch"] = float((final - want).abs().max())
    del want
    torch.cuda.empty_cache()
    out["torch_gpu_ms"] = timed(lambda: re_ranking(qg_d, qq_d, gg_d, k1=k1, k2=k2, lambda_value=lam, device="cuda"),
                                max(1, args.reps // 2))
    if not args.skip_host_torch:
        hq, hd = min(args.host_q, args.n_q), min(args.host_db, args.n_db)
        sub = [torch.from_numpy(qg[:hq, :hd]), torch.from_numpy(qq[:hq, :hq]), torch.from_numpy(gg[:hd, :hd])]
        t0 = time.perf_counter()
        re_ranking(*sub, k1=k1, k2=k2, lambda_value=lam, device="cpu")
        out["torch_host_ms"] = (time.perf_counter() - t0) * 1e3
        out["host_subset"] = [hq, hd]
        out["host_threads"] = torch.get_num_threads()
    out["card"], out["power_limit"], out["sm_clock"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

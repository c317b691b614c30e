#!/usr/bin/env python
"""Measure k-reciprocal re-ranking on sparse data (neighbour pass + sparse stage) on synthetic descriptors.

    python tools/bench_rerank.py --n-q 6816 --n-db 10000 --compare-dense          # Pitts30k-test shape
    python tools/bench_rerank.py --n-q 8280 --n-db 83952                          # Pitts250k-test shape
    python tools/bench_rerank.py --n-q 6800 --n-db 250000 --emulate-world 8       # 8 neighbour-pass slices, 1 GPU
    python -m torch.distributed.run --nproc-per-node 8 tools/bench_rerank.py --n-q 6800 --n-db 250000

Prints one JSON line: CUDA-event times per stage, torch.cuda.max_memory_allocated, the engine's re-ranking
workspace, a hash of the top-k (identical for every world size), how many rows the neighbour pass's guards sent to
the exact scan (emulated mode), and the card name and power limit.
--emulate-world W runs the neighbour pass as W row slices on one GPU, as W ranks would.  With --compare-dense (only
where the [N,N] matrices fit) the dense re_ranking of openibl_b200/utils/rerank.py is timed in the same run and its
top-k compared."""
import argparse
import hashlib
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from openibl_b200 import synth  # noqa: E402
from openibl_b200.engine import Engine  # noqa: E402
from openibl_b200.utils.data.sampler import slice_bounds  # noqa: E402


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                             "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = pl.stdout.strip() or None
    except Exception:
        power = None
    return name, power


def topk_hash(fd, fi):
    h = hashlib.sha256()
    h.update(fi.cpu().numpy().tobytes())
    h.update(fd.cpu().numpy().tobytes())
    return h.hexdigest()[:16]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-q", type=int, default=6816)
    ap.add_argument("--n-db", type=int, default=10000)
    ap.add_argument("--dim", type=int, default=4096)
    ap.add_argument("--k1", type=int, default=20)
    ap.add_argument("--k2", type=int, default=6)
    ap.add_argument("--lambda-value", type=float, default=0.3)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--emulate-world", type=int, default=1)
    ap.add_argument("--compare-dense", action="store_true")
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()

    distributed = int(os.environ.get("WORLD_SIZE", "1")) > 1
    if distributed:
        import torch.distributed as dist
        local = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(local)
        dist.init_process_group("nccl")
        rank, world = dist.get_rank(), dist.get_world_size()
    else:
        rank, world = 0, args.emulate_world
    dev = torch.device("cuda", torch.cuda.current_device())
    eng = Engine.get(dev)
    q, db, _ = synth.make_gallery(n_db=args.n_db, n_q=args.n_q, dim=args.dim)
    q, db = q.to(dev), db.to(dev)
    m, n = q.shape[0], db.shape[0]
    N = m + n
    w = max(args.k1 + 1, args.k2)
    torch.cuda.synchronize()
    base_mem = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()

    def run():
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        if distributed:
            from openibl_b200.evaluators import sharded_rerank_topk
            lo, cnt, _ = slice_bounds(n, world, rank)
            res = sharded_rerank_topk(q, db[lo:lo + cnt], args.k, lo, cnt, args.k1, args.k2, args.lambda_value)
            ev[1].record(); ev[2].record(); ev[3].record()
            return res, ev
        X = torch.cat([q, db])
        parts = []
        for r in range(world):                    # the row slices W ranks would each compute
            lo, cnt, _ = slice_bounds(N, world, r)
            parts.append(eng.knn_rowmax(X, w, lo, cnt))
        idx = torch.cat([p[0] for p in parts])
        dd = torch.cat([p[1] for p in parts])
        mx = torch.cat([p[2] for p in parts])
        ev[1].record()
        orig = None
        if args.lambda_value > 0:
            _, orig = eng.l2dist_topk(q, db, min(args.k + 8, 128, n))
        ev[2].record()
        res = eng.rerank_topk(X, m, idx, dd, mx, args.k1, args.k2, args.lambda_value, args.k, orig)
        ev[3].record()
        return res, ev

    for _ in range(args.warmup):
        run()
    torch.cuda.synchronize()
    res, ev = run()
    torch.cuda.synchronize()
    out = {"n_q": m, "n_db": n, "dim": args.dim, "k1": args.k1, "k2": args.k2, "lambda": args.lambda_value,
           "k": args.k, "world": world, "mode": "nccl" if distributed else "emulated"}
    name, power = card()
    out.update({"gpu": name, "power_limit": power})
    if rank == 0:
        fd, fi = res
        if distributed:
            out["total_ms"] = ev[0].elapsed_time(ev[3])
        else:
            out.update({"knn_ms": ev[0].elapsed_time(ev[1]), "orig_topk_ms": ev[1].elapsed_time(ev[2]),
                        "sparse_ms": ev[2].elapsed_time(ev[3]), "total_ms": ev[0].elapsed_time(ev[3])})
        out["max_memory_allocated_above_inputs"] = torch.cuda.max_memory_allocated() - base_mem
        out["rerank_workspace_bytes"] = eng.rerank_workspace_bytes()
        out["topk_hash"] = topk_hash(fd, fi)
        if not distributed:                   # rows the guards sent to the exact scan, in an untimed pass
            X = torch.cat([q, db])
            flagged = 0
            for r in range(world):
                lo, cnt, _ = slice_bounds(N, world, r)
                eng.knn_rowmax(X, w, lo, cnt)
                flagged += max(eng.knn_flagged(), 0)
            out["knn_exact_scan_rows"] = flagged
            del X
        if args.compare_dense:
            from openibl_b200.utils.rerank import re_ranking
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            final = re_ranking(eng.l2dist_dense(q, db), eng.l2dist_dense(q, q), eng.l2dist_dense(db, db),
                               k1=args.k1, k2=args.k2, lambda_value=args.lambda_value)
            dd_, di_ = eng.topk_rows(final.contiguous(), args.k)
            e1.record()
            torch.cuda.synchronize()
            out["dense_ms"] = e0.elapsed_time(e1)
            out["dense_top1_agree"] = float((di_[:, 0] == fi[:, 0]).float().mean())
            out["dense_topk_index_agree"] = float((di_ == fi).float().mean())
            out["dense_topk_value_maxdiff"] = float((dd_ - fd).abs().max())
        print(json.dumps(out))
    if distributed:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()

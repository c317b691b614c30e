"""Times searches over a prepared database (Engine.search_prepared) against ibl_l2dist_topk on the same rows, and the
streaming scan kernel's share of the HBM bandwidth.

For each database size n x 4096 and query batch (m, k): the median of CUDA-event timings of whole calls after
warm-up, for both entry points, with their outputs asserted identical; then, in a separate profiled run, the device
time of db_scan_dist_kernel alone (torch.profiler), and the fp16 plane bytes (n x d x 2, read once per pass of up to
128 queries) over that time against the 3.35 TB/s of the H100 SXM data sheet.  The card's name, power limit and
maximum SM clock are read in the same run.  Writes one JSON line per configuration to stdout and, with --out, to a
file.  guard_listed counts the queries the screening guard sent to the exact fp32 scan of the whole database.

    python tools/bench_index.py [--d 4096] [--iters 20] [--out results.jsonl]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from openibl_b200.engine import Engine  # noqa: E402

PEAK_BPS = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def time_ms(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def scan_kernel_ms(fn, calls=5):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    total, count = 0.0, 0
    for ev in prof.events():
        if "db_scan_dist_kernel" in ev.name and ev.device_type.name == "CUDA":
            total += ev.device_time
            count += 1
    return (total / 1e3 / calls) if count else float("nan"), count // calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--d", type=int, default=4096)
    ap.add_argument("--n", type=int, nargs="+", default=[10000, 83952, 250000])
    ap.add_argument("--m", type=int, nargs="+", default=[1, 8, 64, 128])
    ap.add_argument("--k", type=int, nargs="+", default=[10, 120])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_index needs a GPU"
    eng = Engine.get(0)
    eng.set_gemm_mode(1)
    info = card()
    print(f"# {info}", flush=True)
    sink = open(args.out, "w") if args.out else None
    g = torch.Generator(device="cuda").manual_seed(0)
    for n in args.n:
        db = torch.nn.functional.normalize(torch.randn(n, args.d, device="cuda", generator=g), dim=1).contiguous()
        prep = eng.prepare_database(db)
        prep_ms = time_ms(lambda: eng.prepare_database(db), 3, warmup=1)
        for m in args.m:
            q = (db[torch.randint(0, n, (m,), device="cuda", generator=g)]
                 + 0.3 * torch.nn.functional.normalize(torch.randn(m, args.d, device="cuda", generator=g), dim=1))
            q = q.contiguous()
            for k in args.k:
                wd, wi = eng.l2dist_topk(q, db, k)
                gd, gi = eng.search_prepared(q, prep, k)
                path, flagged = eng.dist_path(), eng.dist_flagged()
                assert torch.equal(wi, gi) and torch.equal(wd, gd), (n, m, k)
                t_new = time_ms(lambda: eng.search_prepared(q, prep, k), args.iters)
                t_old = time_ms(lambda: eng.l2dist_topk(q, db, k), args.iters)
                kern_ms, _ = scan_kernel_ms(lambda: eng.search_prepared(q, prep, k)) if path == 4 else (None, 0)
                plane = n * args.d * 2 * max(1, -(-m // 128))
                row = {"card": info, "n": n, "d": args.d, "m": m, "k": k, "path": path, "guard_listed": flagged,
                       "search_prepared_ms": round(t_new, 4), "l2dist_topk_ms": round(t_old, 4),
                       "speedup": round(t_old / t_new, 2), "prepare_ms": round(prep_ms, 3),
                       "scan_kernel_ms": None if kern_ms is None else round(kern_ms, 4),
                       "plane_GBps_kernel": None if kern_ms is None else round(plane / kern_ms / 1e6, 1),
                       "share_of_3.35TBps_kernel": None if kern_ms is None else round(plane / kern_ms / 1e-3 / PEAK_BPS, 3),
                       "share_of_3.35TBps_call": round(plane / t_new / 1e-3 / PEAK_BPS, 3)}
                line = json.dumps(row)
                print(line, flush=True)
                if sink:
                    sink.write(line + "\n")
                    sink.flush()
        del prep, db
        torch.cuda.empty_cache()
    if sink:
        sink.close()


if __name__ == "__main__":
    main()

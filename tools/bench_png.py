#!/usr/bin/env python
"""PNGs on the device vs the Pillow fallback; prints one JSON line.

Inputs: a batch of seeded synthetic 480x640 RGB PNGs written by Pillow's encoder at its defaults (zlib level 6, its
own filter choice).  Reports, median of `--reps` after warm-up:
  * `decode_to_tensor` end to end (host parse, H2D, decode, normalise, synchronised) on the device path, and the same
    files through the Pillow fallback (the PNG parse switched off, as before the device decoder existed);
  * the device time of the inflate and unfilter kernels (torch.profiler, one batch);
  * Pillow's per-image decode on this host's CPU.
The card, its power limit and the SM clock after the timed loops are read in the same run.

    python tools/bench_png.py [--batch 32] [--reps 20]
"""
import argparse
import io
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _files(n, h, w, seed):
    from PIL import Image
    out = []
    for i in range(n):
        r = np.random.default_rng(seed + i)
        b0 = r.integers(0, 256, (h // 16 + 2, w // 16 + 2, 3)).astype(np.uint8)
        a = np.asarray(Image.fromarray(b0).resize((w, h), Image.BILINEAR)).astype(np.int16)
        im = Image.fromarray(np.clip(a + r.integers(-12, 13, a.shape), 0, 255).astype(np.uint8))
        b = io.BytesIO()
        im.save(b, "PNG")
        out.append(b.getvalue())
    return out


def _wall(fn, reps, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def _smi(query):
    q = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return [s.strip() for s in q[0].split(",")] if q else ["unknown"] * (query.count(",") + 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    from PIL import Image
    from openibl_b200 import _cabi
    from openibl_b200.engine import Engine
    from openibl_b200.utils.data.gpu_jpeg import decode_to_tensor

    card, power = _smi("name,power.limit")
    B, H, W = args.batch, 480, 640
    files = _files(B, H, W, 2000)
    assert all(_cabi.png_parse(f)["ok"] for f in files)
    eng = Engine.get(0)
    res = {"card": card, "power_limit": power, "batch": B, "size": [H, W],
           "kb_per_image": round(sum(map(len, files)) / B / 1e3, 1)}
    res["device_ms"] = round(_wall(lambda: decode_to_tensor(files, H, W), args.reps), 2)
    real = _cabi.png_parse
    _cabi.png_parse = lambda data: dict(real(data), ok=False)   # the fallback path, as before
    try:
        res["pillow_fallback_ms"] = round(_wall(lambda: decode_to_tensor(files, H, W), args.reps, warm=1), 2)
    finally:
        _cabi.png_parse = real
    res["speedup_vs_fallback"] = round(res["pillow_fallback_ms"] / res["device_ms"], 2)

    from torch.profiler import ProfilerActivity, profile
    decode_to_tensor(files, H, W)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        decode_to_tensor(files, H, W)
        torch.cuda.synchronize()
    kinds = {"inflate": "png_inflate", "unfilter": "png_unfilter", "resize": "resize", "normalise": "u8"}
    ms = {k: 0.0 for k in kinds}
    for ev in p.key_averages():
        for k, pat in kinds.items():
            if pat in ev.key:
                ms[k] += ev.device_time_total / 1e3
    res["kernel_ms"] = {k: round(v, 3) for k, v in ms.items()}

    ts = []
    for _ in range(3):
        t0 = time.perf_counter()
        for f in files:
            np.asarray(Image.open(io.BytesIO(f)).convert("RGB"))
        ts.append((time.perf_counter() - t0) * 1e3 / len(files))
    res["pillow_ms_per_image"] = round(statistics.median(ts), 2)
    res["sm_clock_mhz_after"] = _smi("clocks.sm")[0]
    print(json.dumps(res))


if __name__ == "__main__":
    main()

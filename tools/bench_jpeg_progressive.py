#!/usr/bin/env python
"""Progressive JPEGs on the device vs the Pillow fallback; prints one JSON line.

Inputs: a batch of seeded synthetic 480x640 quality-92 4:2:0 progressive JPEGs (Pillow's `progressive=True`, libjpeg's
simple progression) and their baseline twins (the same image saved without `progressive`).  Reports, median of
`--reps` after warm-up:
  * `decode_to_tensor` end to end (host parse, H2D, decode, normalise, synchronised) for the progressive files on the
    device path, the same files through the Pillow fallback (the device decoder for progressive files switched off, as
    before it existed) and the baseline twins;
  * the device kernel time of every scan kind and of the shared IDCT / colour kernels (torch.profiler, one batch);
  * Pillow's per-image decode of a progressive file and of its twin on this host's CPU.
The card, its power limit and the SM clock after the timed loops are read in the same run.

    python tools/bench_jpeg_progressive.py [--batch 32] [--reps 20]
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


def _pairs(n, h, w, seed):
    from PIL import Image
    prog, base = [], []
    for i in range(n):
        r = np.random.default_rng(seed + i)
        b0 = r.integers(0, 256, (h // 16 + 2, w // 16 + 2, 3)).astype(np.uint8)
        a = np.asarray(Image.fromarray(b0).resize((w, h), Image.BILINEAR)).astype(np.int16)
        im = Image.fromarray(np.clip(a + r.integers(-12, 13, a.shape), 0, 255).astype(np.uint8))
        for out, kw in ((prog, {"progressive": True}), (base, {})):
            b = io.BytesIO()
            im.save(b, "JPEG", quality=92, subsampling=2, **kw)
            out.append(b.getvalue())
    return prog, base


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
    prog, base = _pairs(B, H, W, 1000)
    assert all(_cabi.jpeg_parse_progressive(f)["ok"] for f in prog) and all(_cabi.jpeg_parse(f)["ok"] for f in base)
    eng = Engine.get(0)
    res = {"card": card, "power_limit": power, "batch": B, "size": [H, W], "quality": 92, "subsampling": "4:2:0",
           "progressive_kb_per_image": round(sum(map(len, prog)) / B / 1e3, 1),
           "baseline_kb_per_image": round(sum(map(len, base)) / B / 1e3, 1)}
    res["progressive_device_ms"] = round(_wall(lambda: decode_to_tensor(prog, H, W), args.reps), 2)
    res["baseline_device_ms"] = round(_wall(lambda: decode_to_tensor(base, H, W), args.reps), 2)
    real = _cabi.jpeg_parse_progressive
    _cabi.jpeg_parse_progressive = lambda data: dict(real(data), ok=False)   # the fallback path, as before
    try:
        res["progressive_pillow_fallback_ms"] = round(_wall(lambda: decode_to_tensor(prog, H, W), args.reps, warm=1), 2)
    finally:
        _cabi.jpeg_parse_progressive = real
    res["speedup_vs_fallback"] = round(res["progressive_pillow_fallback_ms"] / res["progressive_device_ms"], 2)

    # device kernel time per scan kind (one batch)
    from torch.profiler import ProfilerActivity, profile
    decode_to_tensor(prog, H, W)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        decode_to_tensor(prog, H, W)
        torch.cuda.synchronize()
    kinds = {"dc_first": "jpeg_prog_dc_first", "dc_refine": "jpeg_prog_dc_refine", "ac_first": "jpeg_prog_ac_first",
             "ac_refine": "jpeg_prog_ac_refine", "idct": "jpeg_idct", "color": "jpeg_color"}
    ms = {k: 0.0 for k in kinds}
    for ev in p.key_averages():
        for k, pat in kinds.items():
            if pat in ev.key:
                ms[k] += ev.device_time_total / 1e3
    res["kernel_ms"] = {k: round(v, 3) for k, v in ms.items()}
    entropy = sum(ms[k] for k in ("dc_first", "dc_refine", "ac_first", "ac_refine"))
    res["entropy_decode_share"] = {k: round(ms[k] / entropy, 3) for k in ("dc_first", "dc_refine", "ac_first",
                                                                         "ac_refine")} if entropy else {}

    def pil(files):
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            for f in files:
                np.asarray(Image.open(io.BytesIO(f)).convert("RGB"))
            ts.append((time.perf_counter() - t0) * 1e3 / len(files))
        return round(statistics.median(ts), 2)
    res["pillow_ms_per_image_progressive"] = pil(prog)
    res["pillow_ms_per_image_baseline"] = pil(base)
    res["sm_clock_mhz_after"] = _smi("clocks.sm")[0]
    print(json.dumps(res))


if __name__ == "__main__":
    main()

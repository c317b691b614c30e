#!/usr/bin/env python
"""Training input side: the device path (JPEG decode + ColorJitter + Resize + ToTensor + Normalize on the GPU, from
file bytes) vs the host train transform; prints one JSON line.

Inputs are seeded synthetic 480x640 JPEGs (quality 92, 4:2:0 like datasets/synthetic.py) and the transform is
`get_transformer_train(480, 640)` of examples/netvlad_img.py's defaults.  Reports
  * the host path per image on one core: Pillow decode + the reference train transform, and ColorJitter alone;
  * the device path for tuple batches of 12, 48 and 88 images (a `netvlad_img.py` step at tuple_size 1 and 4, and an
    SFRS step at tuple_size 4): end to end on the host clock (carriers in, fp32 tensor on the device, synchronised);
    the device time of its kernels and copies, and of the two jitter kernels among them (torch.profiler, separate
    run over fresh decodes); and the jitter call alone on CUDA events, with the decoded pixels restored from a
    pristine copy before every repetition (the jitter works in place, and re-jittering its own output drifts towards
    grey pixels, which skip most of the hue step's arithmetic);
  * H2D bytes per image on each path.
The card name, power limit and SM clock (sampled right after the timed loops) are read in the same run.

    python tools/bench_train_input.py [--reps 20]
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

H, W = 480, 640


def _jpegs(n, seed):
    from PIL import Image
    out = []
    for i in range(n):
        r = np.random.default_rng(seed + i)
        base = r.integers(0, 256, (H // 16 + 2, W // 16 + 2, 3)).astype(np.uint8)
        a = np.asarray(Image.fromarray(base).resize((W, H), Image.BILINEAR)).astype(np.int16)
        a = np.clip(a + r.integers(-12, 13, a.shape), 0, 255).astype(np.uint8)
        b = io.BytesIO()
        Image.fromarray(a).save(b, "JPEG", quality=92)
        out.append(b.getvalue())
    return out


def _events_restored(fn, imgs, reps, warm=3):
    """CUDA events around fn, the in-place images reset to their decoded pixels before every call (outside the events)."""
    pristine = [im.clone() for im in imgs]
    ts = []
    for r in range(warm + reps):
        for im, p in zip(imgs, pristine):
            im.copy_(p)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        if r >= warm:
            ts.append(s.elapsed_time(e))
    return statistics.median(ts)


def _profiled_ms(fn, reps=5):
    """Device time per call of the path's kernels and copies, and of the jitter kernels alone (torch.profiler)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    total = jitter = 0.0
    for ev in prof.key_averages():
        if any(t in ev.key for t in ("jpeg_", "color_jitter_", "resize_", "u8_hwc_to_nchw", "Memcpy", "Memset")):
            t = getattr(ev, "device_time_total", None)
            t = (ev.cuda_time_total if t is None else t) / reps / 1e3
            total += t
            if "color_jitter_" in ev.key:
                jitter += t
    return total, jitter


def _host_clock(fn, reps, warm=3):
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


def _smi(fields):
    q = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return [s.strip() for s in q[0].split(",")] if q else ["unknown"] * len(fields.split(","))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    from PIL import Image
    import torchvision.transforms as T
    from openibl_b200 import _cabi
    from openibl_b200.engine import Engine
    from openibl_b200.utils.data import get_transformer_train
    from openibl_b200.utils.data.gpu_jpeg import decode_batch

    card, power, max_sm = _smi("name,power.limit,clocks.max.sm")
    files = _jpegs(88, 0)
    res = {"card": card, "power_limit": power, "max_sm_clock": max_sm, "image": f"{H}x{W}",
           "jpeg_bytes": int(np.mean([len(f) for f in files]))}

    # host path, one core
    torch.set_num_threads(1)
    host_tf = get_transformer_train(H, W)
    cj = T.ColorJitter(0.7, 0.7, 0.7, 0.5)
    torch.manual_seed(0)
    n = 24
    t0 = time.perf_counter()
    for f in files[:n]:
        host_tf(Image.open(io.BytesIO(f)).convert("RGB"))
    res["host_decode_and_train_transform_ms_per_image"] = (time.perf_counter() - t0) * 1e3 / n
    pils = [Image.open(io.BytesIO(f)).convert("RGB") for f in files[:n]]
    t0 = time.perf_counter()
    for im in pils:
        cj(im)
    res["host_color_jitter_ms_per_image"] = (time.perf_counter() - t0) * 1e3 / n
    torch.set_num_threads(os.cpu_count() or 1)

    infos = [_cabi.jpeg_parse(f) for f in files]
    # destuffed entropy data + 8 pad bytes per interval + tables/descriptors (~9 KB) + the jitter descriptor and sum
    res["h2d_bytes_per_image_device_path"] = int(np.mean([i["entropy_bytes"] + 8 * i["intervals"] for i in infos])
                                                 + 9216 + 64)
    res["h2d_bytes_per_image_host_path"] = H * W * 3 * 4

    eng = Engine.get(0)
    dev_tf = get_transformer_train(H, W, device_decode=True)
    torch.manual_seed(0)
    carriers = [dev_tf(f, f"img{i}.jpg") for i, f in enumerate(files)]
    for b in (12, 48, 88):
        batch = carriers[:b]
        res[f"device_end_to_end_ms_{b}"] = _host_clock(lambda: decode_batch(batch), args.reps)
        res[f"device_end_to_end_ms_per_image_{b}"] = res[f"device_end_to_end_ms_{b}"] / b
        imgs, _ = eng.decode_jpeg_async(batch)
        params = [c.jitter for c in batch]
        res[f"jitter_call_events_ms_{b}"] = _events_restored(lambda: eng.color_jitter_u8(imgs, params), imgs,
                                                             args.reps)
    res["sm_clock_after_timing"] = _smi("clocks.sm")[0]
    for b in (12, 48, 88):                                      # profiled separately: tracing slows the host
        batch = carriers[:b]
        res[f"device_kernels_and_copies_ms_{b}"], res[f"jitter_kernels_profiled_ms_{b}"] = _profiled_ms(
            lambda: decode_batch(batch))
    # the host path's copy of a 48-image stacked fp32 tuple batch (pageable, as _parse_data does it)
    x48 = torch.randn(48, 3, H, W)
    res["host_path_h2d_ms_48"] = _host_clock(lambda: x48.cuda(), args.reps)
    print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in res.items()}))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Device JPEG decode + test transform vs the host transform; prints one JSON line.

Inputs are seeded synthetic JPEGs (quality 92, 4:2:0 like datasets/synthetic.py): a 480x640 set and a 1224x1632 set.
Reports the host transform per image on one core, the device decode + resize + normalise time per batch of 32
(CUDA events, median of 20 after warm-up), per-stage kernel times (torch.profiler, separate run), H2D bytes per image,
extraction images/s at batch 32 from file bytes next to ibl_extract_host_u8 and the fp32 host path, and the
batch-1 latency of a Tokyo-size (1224x1632) image.  The card name and power limit are read in the same run.

    python tools/bench_jpeg.py [--batch 32] [--reps 20]
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


def _jpegs(n, h, w, seed):
    from PIL import Image
    out = []
    for i in range(n):
        r = np.random.default_rng(seed + i)
        base = r.integers(0, 256, (h // 16 + 2, w // 16 + 2, 3)).astype(np.uint8)
        a = np.asarray(Image.fromarray(base).resize((w, h), Image.BILINEAR)).astype(np.int16)
        a = np.clip(a + r.integers(-12, 13, a.shape), 0, 255).astype(np.uint8)
        b = io.BytesIO()
        Image.fromarray(a).save(b, "JPEG", quality=92)
        out.append(b.getvalue())
    return out


def _events(fn, reps, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        e.synchronize()
        ts.append(s.elapsed_time(e))
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    from PIL import Image
    from openibl_b200 import _cabi, synth
    from openibl_b200.engine import Engine
    from openibl_b200.utils.data import _MEAN, _STD, get_transformer_test
    from openibl_b200.utils.data.gpu_jpeg import decode_to_tensor

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    card, power = [s.strip() for s in q[0].split(",")] if q else ("unknown", "unknown")
    B, H, W = args.batch, 480, 640
    small = _jpegs(B, H, W, 0)
    big = _jpegs(B, 1224, 1632, 1000)
    res = {"card": card, "power_limit": power, "batch": B, "jpeg_bytes_480x640": int(np.mean([len(f) for f in small])),
           "jpeg_bytes_1224x1632": int(np.mean([len(f) for f in big]))}

    # host transform, one core
    torch.set_num_threads(1)
    tf = get_transformer_test(H, W)
    t0 = time.perf_counter()
    for f in small:
        tf(Image.open(io.BytesIO(f)).convert("RGB"))
    res["host_transform_ms_per_image_480x640"] = (time.perf_counter() - t0) * 1e3 / B
    t0 = time.perf_counter()
    for f in big[:8]:
        tf(Image.open(io.BytesIO(f)).convert("RGB"))
    res["host_transform_ms_per_image_1224x1632"] = (time.perf_counter() - t0) * 1e3 / 8
    torch.set_num_threads(os.cpu_count() or 1)

    dev = torch.device("cuda", 0)
    eng = Engine.get(0)
    # H2D bytes: destuffed entropy data, 8 pad bytes per interval, six Huffman tables + descriptors (~9 KB)
    infos = [_cabi.jpeg_parse(f) for f in small]
    res["h2d_bytes_per_image_480x640"] = int(np.mean([i["entropy_bytes"] + 8 * i["intervals"] for i in infos]) + 9216)
    res["h2d_bytes_per_image_fp32_host_path"] = H * W * 3 * 4
    res["h2d_bytes_per_image_u8_host_path"] = H * W * 3

    res["device_decode_transform_ms_per_batch_480x640"] = _events(lambda: decode_to_tensor(small, H, W), args.reps)
    res["device_decode_transform_ms_per_batch_1224x1632_to_480x640"] = _events(
        lambda: decode_to_tensor(big, H, W), max(5, args.reps // 4))
    res["device_decode_only_ms_per_batch_480x640"] = _events(lambda: eng.decode_jpeg_async(small), args.reps)
    res["tokyo_1224x1632_batch1_latency_ms"] = _events(lambda: decode_to_tensor(big[:1], H, W, tokyo=True), args.reps)

    # per-stage kernel times (separate, profiled run)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            decode_to_tensor(small, H, W)
        torch.cuda.synchronize()
    stages = {}
    for ev in prof.key_averages():
        name = ev.key
        for tag in ("jpeg_sync", "jpeg_fix", "jpeg_write", "jpeg_dc", "jpeg_idct", "jpeg_color", "resize_h_u8",
                    "resize_v_u8", "u8_hwc_to_nchw", "Memcpy HtoD", "Memset"):
            if tag in name:
                t = getattr(ev, "device_time_total", None)
                if t is None:
                    t = ev.cuda_time_total
                stages[tag] = stages.get(tag, 0.0) + t / 5 / 1e3
    res["stage_ms_per_batch_480x640"] = {k: round(v, 4) for k, v in stages.items()}

    # extraction at batch B: file bytes vs host uint8 vs host fp32
    sd = synth.make_state_dict(seed=5, with_pca=True, pca_dim=4096)
    sdd = {k: v.to(dev) for k, v in sd.items()}
    slots = synth.VGG16_CONV_SLOTS
    eng.set_vgg16([sdd[f"base_model.base.{s}.weight"] for s in slots], [sdd[f"base_model.base.{s}.bias"] for s in slots])
    eng.set_netvlad(sdd["net_vlad.conv.weight"], sdd["net_vlad.centroids"])
    eng.set_pca(sdd["pca_layer.weight"], sdd["pca_layer.bias"])
    u8 = torch.stack([torch.from_numpy(np.array(Image.open(io.BytesIO(f)).convert("RGB"))) for f in small]).pin_memory()
    f32 = torch.stack([tf(Image.open(io.BytesIO(f)).convert("RGB")) for f in small]).contiguous().pin_memory()
    out_host = torch.empty(B, 4096).pin_memory()

    def from_bytes():
        x = decode_to_tensor(small, H, W, pending=[])
        eng.extract(x, pca=True)

    def reps_per_s(fn, n=10):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
        return B * n / (time.perf_counter() - t0)
    res["extract_images_per_s_from_file_bytes"] = reps_per_s(from_bytes)
    res["extract_images_per_s_host_u8"] = reps_per_s(lambda: eng.extract_host_u8(u8, out_host, _MEAN, _STD, pca=True))
    res["extract_images_per_s_host_fp32"] = reps_per_s(lambda: eng.extract_host(f32, out_host, pca=True))
    x = decode_to_tensor(small, H, W)
    res["extract_ms_per_batch_device_input"] = _events(lambda: eng.extract(x, pca=True), 10)
    res["decode_share_of_extraction"] = (res["device_decode_transform_ms_per_batch_480x640"] /
                                         res["extract_ms_per_batch_device_input"])
    print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in res.items()}))


if __name__ == "__main__":
    main()

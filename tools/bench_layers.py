"""Per-layer device times of the VGG16 trunk as the forward runs it, batch 32 at 480x640 (same process, CUDA events):
the fused conv1_1 + conv1_2 + pool kernel, then conv2_1..conv5_3 with their default tiles, so the rows sum to the trunk.
Prints the card, its power limit and the median SM clock sampled during the timed launches.

    python tools/bench_layers.py [--reps 5] [--json OUT.json]
"""
import argparse, ctypes, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from bench import ClockSampler, peaks
from openibl_b200 import synth
from openibl_b200.engine import Engine, _ptr
from openibl_b200._cabi import check

NAMES = ["conv1_1", "conv1_2", "conv2_1", "conv2_2", "conv3_1", "conv3_2", "conv3_3", "conv4_1", "conv4_2", "conv4_3",
         "conv5_1", "conv5_2", "conv5_3"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the table to this file")
    args = ap.parse_args()
    B = args.batch
    eng = Engine.get(0)
    sd = {k: v.cuda() for k, v in synth.make_vgg_weights(0).items()}
    slots = synth.VGG16_CONV_SLOTS
    eng.set_vgg16([sd[f"base.{s}.weight"] for s in slots], [sd[f"base.{s}.bias"] for s in slots])
    shapes, h, w = [], 480, 640
    for item in synth.VGG16_PLAN:
        if item == "P":
            h, w = h // 2, w // 2
        else:
            shapes.append((h, w, item[1], item[2]))
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    pk = peaks()
    # (label, ibl_debug_time_layer index, H, W, Cin, Cout, algorithmic GFLOP, MMA passes per product)
    rows = [("conv1 fused", -1, 480, 640, 3, 64,
             sum(2.0 * B * hh * ww * 9 * ci * co / 1e9 for hh, ww, ci, co in shapes[:2]), None)]
    for li in range(2, len(shapes)):
        hh, ww, ci, co = shapes[li]
        rows.append((NAMES[li], li, hh, ww, ci, co, 2.0 * B * hh * ww * 9 * ci * co / 1e9, 3))
    sampler = ClockSampler(0)
    sampler.start()
    out = []
    for name, li, hh, ww, ci, co, gf, passes in rows:
        x = torch.randn(B, 3, hh, ww, device="cuda") if li < 0 else torch.randn(B, hh, ww, ci, device="cuda").relu_()
        ms = ctypes.c_float()
        check(eng.lib.ibl_debug_time_layer(eng.h, li, _ptr(x), B, hh, ww, 0, args.reps, ctypes.byref(ms)), "time_layer")
        del x
        out.append({"layer": name, "hw": f"{hh}x{ww}", "cin": ci, "cout": co, "ms": ms.value, "alg_tflops": gf / ms.value,
                    "mma_tflops": gf / ms.value * passes if passes else None})
    clocks = sampler.stop()
    print(f"card: {card}; median SM clock {clocks['sm_mhz']} MHz (max {clocks['sm_max_mhz']}); "
          f"peak {pk['bf16_tflops_sustained']:.0f} TFLOP/s bf16 ({pk['src']})")
    print(f"{'layer':12s} {'HxW':>9s} {'Cin':>4s} {'Cout':>4s} {'ms':>8s} {'alg TF/s':>9s} {'MMA TF/s':>9s} {'of peak':>8s}")
    for r in out:
        mma = f"{r['mma_tflops']:9.1f} {r['mma_tflops'] / pk['bf16_tflops_sustained']:8.3f}" if r["mma_tflops"] else f"{'-':>9s} {'-':>8s}"
        print(f"{r['layer']:12s} {r['hw']:>9s} {r['cin']:4d} {r['cout']:4d} {r['ms']:8.3f} {r['alg_tflops']:9.1f} {mma}")
    total = sum(r["ms"] for r in out)
    print(f"trunk (sum of the {len(out)} launches): {total:.3f} ms")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card, "clocks": clocks, "batch": B, "layers": out, "trunk_ms": total}, f, indent=1)


if __name__ == "__main__":
    main()

"""Where the device time of one flagship step goes: the batch-32 480x640 VGG16 + NetVLAD + PCA extraction built as
bench.py builds it (synthetic state dict, two alternating input batches), warmed up, then --steps steps under
torch.profiler with CUDA activities.  Prints every kernel's device time per step and its share of the summed kernel
time, the step time from CUDA events over the same number of steps without the profiler, and the card, its power
limit and the median SM clock sampled during the un-profiled steps.

    python tools/profile_step.py [--steps 10] [--json OUT.json]
"""
import argparse, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from torch.profiler import ProfilerActivity, profile
from bench import BATCH, H, W, ClockSampler
from openibl_b200 import synth
from openibl_b200.engine import Engine


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--top", type=int, default=15, help="kernels to list (the rest are summed in one row)")
    ap.add_argument("--json", default=None, help="also write the table to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profile_step.py needs a CUDA device (an H100): there is nothing to profile without one")
    dev = torch.device("cuda", 0)
    eng = Engine.get(0)
    sd = {k: v.to(dev) for k, v in synth.make_state_dict(seed=0, with_pca=True).items()}
    slots = synth.VGG16_CONV_SLOTS
    eng.set_vgg16([sd[f"base_model.base.{s}.weight"] for s in slots], [sd[f"base_model.base.{s}.bias"] for s in slots])
    eng.set_netvlad(sd["net_vlad.conv.weight"], sd["net_vlad.centroids"])
    eng.set_pca(sd["pca_layer.weight"], sd["pca_layer.bias"])
    xs = [synth.make_images(seed=100 + i, batch=BATCH).to(dev) for i in range(2)]
    for i in range(max(args.warmup, 2)):
        eng.extract(xs[i % 2], pca=True)
    torch.cuda.synchronize()

    # step time without the profiler
    sampler = ClockSampler(0)
    sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(args.steps):
        eng.extract(xs[i % 2], pca=True)
    e1.record()
    torch.cuda.synchronize()
    clocks = sampler.stop()
    step_ms = e0.elapsed_time(e1) / args.steps

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.steps):
            eng.extract(xs[i % 2], pca=True)
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        us = getattr(e, "self_device_time_total", 0.0)
        if us > 0 and e.device_type == torch.autograd.DeviceType.CUDA:
            k = kernels.setdefault(e.key, [0.0, 0])
            k[0] += us
            k[1] += e.count
    busy_ms = sum(v[0] for v in kernels.values()) / 1e3 / args.steps
    rows = sorted(({"kernel": name, "ms_per_step": us / 1e3 / args.steps, "launches_per_step": n / args.steps,
                    "share_of_kernel_time": us / 1e3 / args.steps / busy_ms} for name, (us, n) in kernels.items()),
                  key=lambda r: -r["ms_per_step"])

    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {card}; median SM clock {clocks['sm_mhz']} MHz (max {clocks['sm_max_mhz']}); "
          f"throttle reasons {clocks['reasons']}")
    print(f"step {step_ms:.3f} ms (CUDA events, {args.steps} steps, no profiler); kernel time {busy_ms:.3f} ms per "
          f"profiled step")
    print(f"{'ms/step':>8s} {'share':>6s} {'launch':>6s}  kernel")
    for r in rows[:args.top]:
        print(f"{r['ms_per_step']:8.3f} {100 * r['share_of_kernel_time']:5.1f}% {r['launches_per_step']:6.1f}  "
              f"{r['kernel'][:110]}")
    rest = rows[args.top:]
    if rest:
        ms = sum(r["ms_per_step"] for r in rest)
        print(f"{ms:8.3f} {100 * ms / busy_ms:5.1f}%         ({len(rest)} other kernels)")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card, "clocks": clocks, "batch": BATCH, "height": H, "width": W, "steps": args.steps,
                       "step_ms": step_ms, "kernel_ms_per_step": busy_ms, "kernels": rows}, f, indent=1)


if __name__ == "__main__":
    main()

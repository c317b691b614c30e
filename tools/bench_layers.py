"""Per-layer device times of the VGG16 backbone at batch 32, 480x640 (same process, CUDA events):
conv1_1 and conv1_2..conv5_3 on the tensor cores (wgmma), the latter with each admissible N tile."""
import ctypes, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from openibl_b200 import synth
from openibl_b200.engine import Engine, _ptr
from openibl_b200._cabi import check

B = int(os.environ.get("B", 32))
eng = Engine.get(0)
sd = {k: v.cuda() for k, v in synth.make_vgg_weights(0).items()}
slots = synth.VGG16_CONV_SLOTS
eng.set_vgg16([sd[f"base.{s}.weight"] for s in slots], [sd[f"base.{s}.bias"] for s in slots])
layers = [p for p in synth.VGG16_PLAN if p != "P"]
shapes, h, w = [], 480, 640
for item in synth.VGG16_PLAN:
    if item == "P":
        h, w = h // 2, w // 2
    else:
        shapes.append((h, w, item[1], item[2]))
peak = json.load(open("MEASURED_PEAKS.json"))["bf16_tflops_sustained"] if os.path.exists("MEASURED_PEAKS.json") else 1451.3
tot = {}
print(f"{'layer':8s} {'HxW':>9s} {'Cin':>4s} {'Cout':>4s} {'BN':>4s} {'ms':>8s} {'alg TF/s':>9s} {'MMA TF/s':>9s} {'of sustained':>12s}")
for li, (hh, ww, cin, cout) in enumerate(shapes):
    if li == 0:
        x = torch.randn(B, 3, hh, ww, device="cuda")
        bns = [0]
    else:
        x = torch.randn(B, hh, ww, cin, device="cuda").relu_()
        bns = [b for b in (64, 128) if cout % b == 0]
    gf = 2.0 * B * hh * ww * 9 * cin * cout / 1e9
    for bn in bns:
        ms = ctypes.c_float()
        check(eng.lib.ibl_debug_time_layer(eng.h, li, _ptr(x), B, hh, ww, cin if False else bn, 5, ctypes.byref(ms)), "time_layer")
        tf = gf / ms.value
        mma = tf * (1 if li == 0 else 3)
        print(f"conv#{li:<3d} {hh:4d}x{ww:<4d} {cin:4d} {cout:4d} {bn:4d} {ms.value:8.3f} {tf:9.1f} {mma:9.1f} {mma/peak:12.3f}")
        tot.setdefault(li, []).append((ms.value, bn))
    del x
best = sum(min(v)[0] for v in tot.values())
dflt = sum(next((m for m, b in v if b == (0 if li == 0 else (128 if shapes[li][3] % 128 == 0 else 64))), v[0][0]) for li, v in tot.items())
print(f"sum default {dflt:.3f} ms   sum best-per-layer {best:.3f} ms   choices {[min(v)[1] for v in tot.values()]}")

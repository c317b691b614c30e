#!/usr/bin/env python
"""Times Engine.l2dist_topk (BASELINE configs[2] shape by default) with CUDA events."""
import os, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from openibl_b200 import synth
from openibl_b200.engine import Engine

m, n, d, k = (int(a) for a in (sys.argv[1:5] if len(sys.argv) >= 5 else (6800, 10000, 4096, 10)))
eng = Engine.get(0)
q, db, gt = synth.make_gallery(n, m, d)
qd, dbd = q.cuda(), db.cuda()
for _ in range(3):
    eng.l2dist_topk(qd, dbd, k)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
reps = 10
e0.record()
for _ in range(reps):
    dk, ik = eng.l2dist_topk(qd, dbd, k)
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / reps
exact = 2 - 2 * (qd[::97].double() @ dbd.double().t())
wi = exact.topk(k, largest=False).indices
print(json.dumps({"m": m, "n": n, "d": d,
                  "ms": ms, "pairs_per_s": m * n / ms * 1e3, "algorithmic_tflops": 2.0 * m * n * d / ms / 1e9,
                  "agree_fp64_subset": float((ik[::97] == wi).float().mean()), "flagged": eng.dist_flagged()}), flush=True)

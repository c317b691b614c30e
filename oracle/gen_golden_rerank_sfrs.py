#!/usr/bin/env python
"""Golden vectors for the SFRS sampler refresh's re-ranking call (examples/netvlad_img_sfrs.py:84): the UNMODIFIED
reference function ibl/utils/rerank.py:32-100 on seeded q-g / q-q / g-g distance matrices.
TEST INFRASTRUCTURE; build container only (needs /root/reference).

    python oracle/gen_golden_rerank_sfrs.py     # writes tests/golden/rerank_sfrs.npz

Cases (name: m, n, d, k1, k2, lambda):
  sfrs   the driver's parameters (k1 = 20, k2 = 1, lambda = 0.1) at a few hundred rows
  k2     k2 = 6, lambda = 0.3
  asym   q-q and g-g scaled entry by entry by 1 + 1e-3 u (u uniform in [-1, 1)), so D[i][j] != D[j][i]: the reference
         reads column i of D for its row i, and a row-reading implementation ranks differently
  tiny   N = m + n = k1 + 1
"""
import importlib.util
import os

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("IBL_REFERENCE", "/root/reference")
spec = importlib.util.spec_from_file_location("ref_rerank", os.path.join(REF, "ibl", "utils", "rerank.py"))
ref = importlib.util.module_from_spec(spec)
spec.loader.exec_module(ref)


def dist(x, y):   # the arithmetic of pairwise_distance (evaluators.py:127-129), fp32
    m, n = x.size(0), y.size(0)
    d = x.pow(2).sum(1, keepdim=True).expand(m, n) + y.pow(2).sum(1, keepdim=True).expand(n, m).t()
    return d.addmm(x, y.t(), beta=1, alpha=-2)


out = {}
cases = [("sfrs", 120, 280, 32, 20, 1, 0.1), ("k2", 60, 200, 24, 20, 6, 0.3), ("asym", 40, 100, 16, 10, 1, 0.3),
         ("tiny", 5, 16, 16, 20, 1, 0.3)]
for ci, (name, m, n, d, k1, k2, lam) in enumerate(cases):
    g = torch.Generator().manual_seed(1000 + ci)
    clusters = max(2, (m + n) // 15)
    centers = torch.randn(clusters, d, generator=g)
    db = torch.nn.functional.normalize(centers[torch.randint(0, clusters, (n,), generator=g)]
                                       + 0.35 * torch.randn(n, d, generator=g), dim=1)
    q = torch.nn.functional.normalize(centers[torch.randint(0, clusters, (m,), generator=g)]
                                      + 0.35 * torch.randn(m, d, generator=g), dim=1)
    qg, qq, gg = dist(q, db), dist(q, q), dist(db, db)
    if name == "asym":
        qq = qq * (1 + 1e-3 * (2 * torch.rand(m, m, generator=g) - 1))
        gg = gg * (1 + 1e-3 * (2 * torch.rand(n, n, generator=g) - 1))
        assert not torch.equal(qq, qq.t()) and not torch.equal(gg, gg.t())
    final = ref.re_ranking(qg.numpy().copy(), qq.numpy().copy(), gg.numpy().copy(), k1=k1, k2=k2, lambda_value=lam)
    out.update({f"{name}_qg": qg.numpy(), f"{name}_qq": qq.numpy(), f"{name}_gg": gg.numpy(),
                f"{name}_final": final.astype(np.float32), f"{name}_params": np.array([k1, k2, lam], dtype=np.float64)})
path = os.path.join(ROOT, "tests", "golden", "rerank_sfrs.npz")
np.savez_compressed(path, **out)
print("wrote", path, os.path.getsize(path) // 1024, "KiB")

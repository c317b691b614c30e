"""BASELINE configs[3]: a Pitts250k-shaped synthetic gallery sharded over the GPUs of one box.

Shared by bench.py (`strong_250k`), tools/bench_gallery.py and tests/test_gpu_e2e_api.py.

Every image is generated on the device from a seed that depends only on its GLOBAL index, so the gallery --
and therefore every descriptor, every distance and the final ranking -- is the same whatever the world
size.  Query j is a noisy copy of database image pos[j] (so Recall@N is a real number); images are smooth random
fields, not white noise.  A random-init trunk still maps all of them to almost the same descriptor (pairwise distances
~1e-5 (tools/diag_gallery.py shows it) -- every query then trips the screening guard and even fp32 "exact"
distances are rounding noise), so callers that want a meaningful ranking first centre the PCA layer on a database sample
(center_pca below: what a PCA fit does); distances are then ~0.8 and Recall@1 goes from 0.999 (query noise 0.1 sigma) to
~0 (0.5 sigma) on 30k images, and 0.2 sigma gives 0.0096 on 250k; the default noise is 0.1 sigma.

Flow (SURVEY 5 / 8e; reference: ibl/evaluators.py:76-101,105-130,142-167 is what it replaces):
  1. rank r extracts its DistributedSliceSampler slice of the database and of the queries
     (ceil(n/W) images, VGG16 + NetVLAD + PCA) -- descriptors stay in that GPU's HBM;
  2. the queries are all-gathered (n_q x 16 KiB);
  3. every rank ranks all queries against its slice (tensor-core distance + top-k + exact re-scoring);
  4. ONE all-gather of the [n_q, k] candidates (8 B each) + a merge kernel.
`emulate_world=W` plays all W ranks on one GPU, one after the other, with the very same slicing and
batching (merge through ibl_topk_merge instead of NCCL): it is how a 1-GPU box checks that the W-GPU
ranking is identical to the 1-GPU ranking.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.distributed as dist

from .evaluators import recalls_from_topk, sharded_topk, _all_gather_rows
from .utils.data.sampler import slice_bounds

import os

SEED_DB, SEED_Q, SEED_POS = 1_000_003, 7_000_003, 12345
NOISE, AMP = float(os.environ.get("IBL_GALLERY_NOISE", 0.1)), 2.0


def planted_positives(n_db: int, n_q: int) -> np.ndarray:
    return np.random.RandomState(SEED_POS).randint(0, n_db, size=n_q)


def make_image_batch(kind: str, first: int, count: int, H: int, W: int, dev, pos=None, out=None) -> torch.Tensor:
    """Images [count,3,H,W] with global indices first..first+count-1; `kind` is 'db' or 'q'.

    A database image is a smooth random field (a 3 x H/16 x W/16 normal sample, seeded by the image's global index,
    bilinearly upsampled and scaled by 2): white noise would give every image almost the same descriptor through a
    random-init trunk (all pairwise distances ~1e-6), smooth structure gives distances of 2e-2..7e-2.  Query j is the
    field of database image pos[j] plus NOISE-sigma white noise seeded by j."""
    x = out if out is not None else torch.empty(count, 3, H, W, device=dev)
    g = torch.Generator(device=dev)
    ch, cw = max(H // 16, 2), max(W // 16, 2)
    for j in range(count):
        i = first + j
        base = i if kind == "db" else int(pos[i])
        g.manual_seed(SEED_DB + base)
        coarse = torch.randn(1, 3, ch, cw, device=dev, generator=g)
        x[j] = torch.nn.functional.interpolate(coarse, size=(H, W), mode="bilinear", align_corners=False)[0] * AMP
        if kind == "q":
            g.manual_seed(SEED_Q + i)
            x[j].add_(torch.randn(3, H, W, device=dev, generator=g), alpha=NOISE)
    return x[:count]


def center_pca(eng, weight: torch.Tensor, H: int, W: int, batch: int, n_sample: int = 256) -> torch.Tensor:
    """Sets the PCA layer's bias to -W.mean, mean = the mean VLAD descriptor of the first `n_sample` database images
    -- what a PCA FIT does (ibl/pca.py:30-33, 86-90 centre the training descriptors; the reference's Conv2d bias is
    -W.mean), without which a random-init trunk's descriptors all point the same way (pairwise distances ~1e-5, the
    ranking then decided by the noise of whatever arithmetic computes them).  Every rank runs this on the SAME images,
    and extraction is batch-invariant, so all ranks set bit-identical parameters.  Returns the bias it set."""
    dev = torch.device("cuda", eng.device)
    acc = None
    buf = torch.empty(batch, 3, H, W, device=dev)
    for b0 in range(0, n_sample, batch):
        nb = min(batch, n_sample - b0)
        v, _ = eng.extract(make_image_batch("db", b0, nb, H, W, dev, out=buf), pca=False)
        acc = v.double().sum(0) if acc is None else acc + v.double().sum(0)
    mean = acc / n_sample
    w2 = weight.detach().reshape(weight.shape[0], -1).to(dev)
    bias = (-(w2.double() @ mean)).float().contiguous()
    eng.set_pca(weight, bias, force=True)
    return bias


def extract_slice(eng, kind: str, n_total: int, world: int, rank: int, H: int, W: int, batch: int, dev, pos=None,
                  pca=True, dim=4096):
    """Descriptors of rank's slice: ([per, dim] GPU tensor with wrap-around padding rows zeroed, lo, cnt, per)."""
    lo, cnt, per = slice_bounds(n_total, world, rank)
    out = torch.zeros(max(per, 1), dim, device=dev)
    buf = torch.empty(batch, 3, H, W, device=dev)
    for b0 in range(0, cnt, batch):
        nb = min(batch, cnt - b0)
        x = make_image_batch(kind, lo + b0, nb, H, W, dev, pos=pos, out=buf)
        d, _ = eng.extract(x, pca=pca)
        out[b0:b0 + nb] = d
    return out, lo, cnt, per


def index_hash(idx: torch.Tensor) -> int:
    """Order-sensitive 63-bit hash of an int64 index tensor (wrapping int64 arithmetic on the device)."""
    flat = idx.reshape(-1).to(torch.int64)
    w = (torch.arange(flat.numel(), device=flat.device, dtype=torch.int64) * 2 + 1) * 0x9E3779B1
    return int(((flat + 1) * w).sum().item()) & 0x7FFFFFFFFFFFFFFF


def exact_subset_agreement(q: torch.Tensor, shard: torch.Tensor, cnt: int, lo: int, k: int, got_idx: torch.Tensor,
                           step: int = 97):
    """fp64 check of a query subset against this shard: fraction of the exact per-shard top-k that appears in
    the engine's top-k candidates of the same shard (near-ties at 1e-7 may swap ranks, never membership by more
    than the last place)."""
    sel = torch.arange(0, q.shape[0], step, device=q.device)
    best = None
    qd = q[sel].double()
    for c0 in range(0, cnt, 32768):
        c1 = min(cnt, c0 + 32768)
        d = 2 - 2 * (qd @ shard[c0:c1].double().t())
        dk, ik = d.topk(min(k, c1 - c0), largest=False)
        ik = ik + c0 + lo
        if best is None:
            best = (dk, ik)
        else:
            dd, ii = torch.cat([best[0], dk], 1), torch.cat([best[1], ik], 1)
            o = dd.argsort(dim=1, stable=True)[:, :k]
            best = (dd.gather(1, o), ii.gather(1, o))
    want = best[1]
    return float((want == got_idx[sel][:, : want.shape[1]]).float().mean())


def run(eng, n_db: int, n_q: int, H: int = 480, W: int = 640, batch: int = 32, k: int = 10, emulate_world: int = 0,
        check_exact: bool = True):
    """Runs the flow above.  Returns a dict (identical on every rank for the ranking fields)."""
    dev = torch.device("cuda", eng.device)
    real_world = dist.get_world_size() if dist.is_initialized() else 1
    real_rank = dist.get_rank() if dist.is_initialized() else 0
    pos = planted_positives(n_db, n_q)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]

    def barrier():
        if real_world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    agree = None
    if emulate_world:
        assert real_world == 1, "emulate_world plays all ranks in ONE process"
        W_ = emulate_world
        barrier()
        ev[0].record()
        shards = [extract_slice(eng, "db", n_db, W_, r, H, W, batch, dev) for r in range(W_)]
        qparts = [extract_slice(eng, "q", n_q, W_, r, H, W, batch, dev, pos=pos) for r in range(W_)]
        ev[1].record()
        q = torch.cat([p[0][: p[3]] for p in qparts])[:n_q].contiguous()
        ev[2].record()
        cands = [eng.l2dist_topk(q, s, k, idx_base=lo, n_valid=cnt) for (s, lo, cnt, per) in shards]
        dk, ik = eng.topk_merge(torch.stack([c[0] for c in cands]), torch.stack([c[1] for c in cands]), k) \
            if W_ > 1 else cands[0]
        ev[3].record()
        world = W_
        if check_exact:
            s, lo, cnt, per = shards[0]
            agree = exact_subset_agreement(q, s, cnt, lo, k, cands[0][1])
    else:
        world = real_world
        barrier()
        ev[0].record()
        shard, lo, cnt, per = extract_slice(eng, "db", n_db, world, real_rank, H, W, batch, dev)
        qslice, _, _, per_q = extract_slice(eng, "q", n_q, world, real_rank, H, W, batch, dev, pos=pos)
        ev[1].record()
        q = _all_gather_rows(qslice[:per_q], per_q)[:n_q].contiguous()
        ev[2].record()
        dk, ik = sharded_topk(q, shard, k, idx_base=lo, n_valid=cnt)
        ev[3].record()
        if check_exact:
            cd, ci = eng.l2dist_topk(q, shard, k, idx_base=lo, n_valid=cnt)
            agree = exact_subset_agreement(q, shard, cnt, lo, k, ci)
    torch.cuda.synchronize()
    t = torch.tensor([ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), ev[2].elapsed_time(ev[3]),
                      ev[0].elapsed_time(ev[3])], device=dev)
    if real_world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        if agree is not None:
            a = torch.tensor([agree], device=dev)
            dist.all_reduce(a, op=dist.ReduceOp.MIN)
            agree = float(a.item())
    ext_ms, gather_ms, rank_ms, total_ms = [float(v) for v in t.tolist()]
    gallery = [("db/%07d" % i, i, 0.0, 0.0) for i in range(n_db)]
    gt = [np.array([int(p)]) for p in pos]
    recalls = recalls_from_topk(ik.cpu().numpy(), gt, gallery)
    sane = bool((ik >= 0).all() and (ik < n_db).all() and (dk[:, 1:] >= dk[:, :-1]).all())
    return {
        "workload": f"{n_db} db + {n_q} query images {H}x{W}, VGG16+NetVLAD+PCA4096, top-{k}, "
                    f"{world} {'emulated ' if emulate_world else ''}GPU(s), db shard {slice_bounds(n_db, world, 0)[2]} rows/GPU",
        "n_gpus": world, "emulated": bool(emulate_world),
        "extract_s": ext_ms / 1e3, "query_allgather_ms": gather_ms, "ranking_ms": rank_ms, "total_s": total_ms / 1e3,
        "images_per_s": (n_db + n_q) / (ext_ms / 1e3), "pairs_per_s": n_q * n_db / (rank_ms / 1e3),
        "recalls": [float(r) for r in recalls], "topk_index_hash": index_hash(ik),
        "topk_dist_checksum": float(dk.double().sum().item()), "topk_sane": sane,
        "exact_fp64_subset_agreement": agree,
    }

"""Host-side mirror of ibl/evaluators.py (reference lines cited per function).

Same call signatures and return types, different data flow:
  * extract_features keeps descriptors on the GPU for the whole loop (one D2H at the end, not one
    per batch, evaluators.py:58) and gathers across ranks with one all_gather;
  * Evaluator.evaluate never builds the [m,n] distance matrix: every rank ranks all queries
    against its own contiguous database slice with the fused distance+top-k kernel, the per-shard
    top-k candidates are all-gathered (NCCL over NVLink) and merged (SURVEY 8e);
  * pairwise_distance still returns the dense matrix for the training callers that need a full
    argsort (netvlad_img.py:78), computed on the GPU.
"""
from __future__ import annotations

import math
import time
from collections import OrderedDict

import numpy as np
import torch
import torch.distributed as dist

from .engine import Engine
from .utils.data.gpu_jpeg import check_decode_errors, decode_batch, is_encoded_batch
from .utils.data.sampler import slice_bounds

__all__ = ["extract_cnn_feature", "extract_features", "pairwise_distance", "spatial_nms",
           "evaluate_all", "recalls_from_topk", "sharded_topk", "gather_merge_topk", "sharded_rerank_topk", "Evaluator"]


def _rank_world():
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def _to_torch(x):
    if torch.is_tensor(x):
        return x
    if type(x).__module__ == "numpy":
        return torch.from_numpy(x)
    raise ValueError("Cannot convert {} to torch tensor".format(type(x)))


def extract_cnn_feature(model, inputs, vlad=True, gpu=None):
    """evaluators.py:22-34: forward, pick vlad/pooled output, L2 (idempotent for vlad).
    A batch of file bytes (get_transformer_test(..., device_decode=True)) is decoded and transformed on the GPU
    first (utils/data/gpu_jpeg.py)."""
    model.eval()
    if is_encoded_batch(inputs):
        inputs = decode_batch(inputs, device=gpu)
    inputs = _to_torch(inputs).cuda(gpu, non_blocking=True)
    with torch.no_grad():
        outputs = model(inputs)
    if isinstance(outputs, (list, tuple)):
        x_pool, x_vlad = outputs
        outputs = x_vlad if vlad else x_pool
    return Engine.get(outputs.device).l2_normalize_rows(outputs)


def _extract_local(model, data_loader, print_freq=10, vlad=True, pca=None, gpu=None):
    """The loop body of extract_features (evaluators.py:51-63) for this rank's slice: returns the descriptors
    as ONE GPU tensor [n_local, D] in loader order plus the file names the loader yielded.  No per-batch
    device->host copy and no synchronisation (the reference does `outputs.data.cpu()` every batch, :58)."""
    model.eval()
    rank, _ = _rank_world()
    if pca is not None:
        pca.load(gpu=gpu)
    feats, names = [], []
    decode_errors = []                   # device JPEG decode: error words, checked once before returning
    end = time.time()
    bt_sum = 0.0
    with torch.no_grad():
        for i, (imgs, fnames, _, _, _) in enumerate(data_loader):
            if is_encoded_batch(imgs):   # file bytes: decode on the GPU, corrupt-file check deferred to the end
                imgs = decode_batch(imgs, device=gpu, pending=decode_errors)
            out = extract_cnn_feature(model, imgs, vlad, gpu=gpu)
            if pca is not None:
                out = pca.infer(out)
            feats.append(out)            # stays on the GPU
            names.extend(fnames)
            bt = time.time() - end
            bt_sum += bt
            end = time.time()
            if (i + 1) % print_freq == 0 and rank == 0:
                print("Extract Features: [{}/{}]\tTime {:.3f} ({:.3f})".format(
                    i + 1, len(data_loader), bt, bt_sum / (i + 1)))
    check_decode_errors(decode_errors)
    if feats:
        return torch.cat(feats), names
    return torch.empty(0, 0, device=torch.device("cuda", torch.cuda.current_device() if gpu is None else gpu)), names


def _all_gather_rows(local, per):
    """[n_local<=per, D] on every rank -> [world*per, D] (rank-major), one NCCL all-gather on device memory."""
    _, world = _rank_world()
    if world == 1:
        return local
    if local.shape[0] != per:
        pad = torch.zeros(per, local.shape[1], device=local.device, dtype=local.dtype)
        pad[: local.shape[0]] = local
        local = pad
    out = torch.empty(world * per, local.shape[1], device=local.device, dtype=local.dtype)
    dist.all_gather_into_tensor(out, local.contiguous())
    return out


def extract_features(model, data_loader, dataset, print_freq=10, vlad=True, pca=None, gpu=None,
                     sync_gather=False):
    """evaluators.py:36-103 -> OrderedDict{fname: CPU FloatTensor[D]} in `dataset` order.
    The loader yields (imgs, fnames, pids, x, y); rank r holds the r-th contiguous padded slice
    (DistributedSliceSampler, sampler.py:194-223).  This is the dict-returning contract the training
    callers and examples/test.py's PCA fit need; Evaluator.evaluate does NOT go through it (shard-resident
    path below)."""
    local, _ = _extract_local(model, data_loader, print_freq, vlad, pca, gpu)
    _, world = _rank_world()
    per = int(math.ceil(len(dataset) * 1.0 / world)) if world > 1 else local.shape[0]
    allf = _all_gather_rows(local, per)
    allf = allf[: len(dataset)].cpu()      # drop the sampler's wrap-around padding; ONE device->host copy
    features = OrderedDict()
    for item, row in zip(dataset, allf):
        features[item[0]] = row
    return features


def pairwise_distance(features, query=None, gallery=None, metric=None):
    """evaluators.py:105-130 -> (dist_m [m,n] CPU tensor, x.numpy(), y.numpy()); the self-distance
    branch (:106-114) when both lists are None.  The GEMM runs on the GPU."""
    eng = Engine.get()
    dev = torch.device("cuda", eng.device)
    if query is None and gallery is None:
        x = torch.stack(list(features.values())).view(len(features), -1)
        if metric is not None:
            x = metric.transform(x)
        xg = x.to(dev)
        return eng.l2dist_self(xg).cpu(), None, None   # 2|x_i|^2 - 2 x_i.x_j, as the reference (:110-113)
    x = torch.stack([features[f] for f, _, _, _ in query]).view(len(query), -1)
    y = torch.stack([features[f] for f, _, _, _ in gallery]).view(len(gallery), -1)
    if metric is not None:
        x = metric.transform(x)
        y = metric.transform(y)
    d = eng.l2dist_dense(x.to(dev), y.to(dev))
    return d.cpu(), x.numpy(), y.numpy()


def spatial_nms(pred, db_ids, topN):
    """evaluators.py:132-140: first occurrence of each place id among the first topN."""
    kept, seen = [], set()
    for p in pred[:topN]:
        pid = db_ids[p]
        if pid not in seen:
            seen.add(pid)
            kept.append(p)
    return kept


def recalls_from_topk(topk_idx, gt, gallery, recall_topk=(1, 5, 10), nms=False):
    """The recall loop of evaluate_all (evaluators.py:151-162) on a [m,k] ranking."""
    topk_idx = np.asarray(topk_idx)
    db_ids = [db[1] for db in gallery]
    correct = np.zeros(len(recall_topk))
    for q, pred in enumerate(topk_idx):
        pred = pred[pred >= 0]
        if nms:
            seen, kept = set(), []
            for p in pred[: max(recall_topk) * 12]:
                pid = db_ids[p]
                if pid not in seen:
                    seen.add(pid)
                    kept.append(p)
            pred = np.asarray(kept, dtype=np.int64)
        for i, n in enumerate(recall_topk):
            if np.any(np.isin(pred[:n], gt[q])):
                correct[i:] += 1
                break
    return correct / len(gt)


def evaluate_all(distmat, gt, gallery, recall_topk=[1, 5, 10], nms=False):
    """evaluators.py:142-167 from a dense matrix; only the consumed ranks are selected (on the GPU)."""
    rank, _ = _rank_world()
    k = max(recall_topk) * (12 if nms else 1)
    d = _to_torch(distmat).float()
    eng = Engine.get()
    k = min(k, d.shape[1])
    if k > 1024:
        # the reference argsorts the whole row and so accepts any recall_topk; the selection kernel keeps
        # up to 1024 ranks per query (Tokyo nms needs 120) -- fail loudly rather than score an empty ranking
        raise NotImplementedError(
            f"evaluate_all needs the first {k} ranks per query; ibl_topk_rows supports at most 1024")
    d = d.to(torch.device("cuda", eng.device))
    _, order = eng.topk_rows(d, k)
    order = order.cpu().numpy()
    recalls = recalls_from_topk(order, gt, gallery, recall_topk, nms)
    if rank == 0:
        print("Recall Scores:")
        for i, kk in enumerate(recall_topk):
            print("  top-{:<4}{:12.1%}".format(kk, recalls[i]))
    return recalls


def sharded_topk(q: torch.Tensor, db_shard: torch.Tensor, k: int, idx_base: int, n_valid: int,
                 _rank_fn=None, _merge_fn=None):
    """Distance + top-k of all queries against this rank's database slice, ONE all-gather of the [m,k]
    candidates, k-way merge.  Returns (dist [m,k], idx [m,k]), identical on every rank.

    The candidates cross NVLink packed as (fp32 distance bits, int32 global index) = 8 bytes each
    (all_gather_into_tensor into one preallocated buffer: 0.54 MB per rank at 6.8k queries, k = 10).
    `_rank_fn` / `_merge_fn` exist only so the gloo CPU test can drive the distributed plumbing without a
    GPU; the product path is the CUDA engine."""
    _, world = _rank_world()
    if _rank_fn is None:
        eng = Engine.get(q.device)
        _rank_fn = lambda qq, dd, kk, base, nv: eng.l2dist_topk(qq, dd, kk, idx_base=base, n_valid=nv)
        _merge_fn = eng.topk_merge
    cd, ci = _rank_fn(q, db_shard, k, idx_base, n_valid)
    if world > 1 and int(idx_base) + int(db_shard.shape[0]) >= 2 ** 31:
        raise ValueError("sharded_topk packs global indices as int32: the gallery must have < 2^31 rows")
    return gather_merge_topk(cd, ci, k, _merge_fn)


def gather_merge_topk(cd: torch.Tensor, ci: torch.Tensor, k: int, merge_fn):
    """This rank's [m,k] candidates (distance, global index) -> the merged [m,k] over all ranks, identical on every
    rank: ONE all_gather_into_tensor of the candidates packed as (fp32 distance bits, int32 index), 8 bytes each,
    then merge_fn(dist [world,m,k], idx [world,m,k], k)."""
    _, world = _rank_world()
    if world == 1:
        return cd, ci
    m = cd.shape[0]
    packed = torch.empty(m, k, 2, dtype=torch.int32, device=cd.device)
    packed[..., 0] = cd.contiguous().view(torch.int32)
    packed[..., 1] = ci                                   # -1 (no candidate) survives the narrowing
    gathered = torch.empty(world * m, k, 2, dtype=torch.int32, device=cd.device)   # rank-major concatenation
    dist.all_gather_into_tensor(gathered, packed)
    gathered = gathered.view(world, m, k, 2)
    gd = gathered[..., 0].contiguous().view(torch.float32)
    gi = gathered[..., 1].to(torch.int64)
    return merge_fn(gd, gi, k)


def sharded_rerank_topk(x: torch.Tensor, shard: torch.Tensor, k: int, idx_base: int, n_valid: int, k1: int = 20,
                        k2: int = 6, lambda_value: float = 0.3):
    """k-reciprocal re-ranking (rerank.py:32-100) of all queries against the sharded gallery, top k only.

    X = [queries; gallery] is assembled on every rank (the gallery takes one device all-gather); each rank runs the
    neighbour pass (first max(k1+1, k2) neighbours by squared distance, exact row maxima) for its slice of the N rows;
    the packed lists (int32 index, fp32 distance bits, and the row maximum: 8 w + 4 bytes per row) take one
    all-gather; rank 0 runs the sparse stage.  Returns (final [m,k], gallery index [m,k]) on rank 0 and None on the
    other ranks.  Nothing of size [m,n] or [N,N] is built, and the result does not depend on the world size."""
    rank, world = _rank_world()
    m = x.shape[0]
    n = int(n_valid)
    if world > 1:
        t = torch.tensor([n], dtype=torch.int64, device=x.device)
        dist.all_reduce(t)
        n = int(t.item())
    N = m + n
    w = max(k1 + 1, k2)
    if N < k1 + 1:
        raise ValueError("re-ranking needs at least k1 + 1 images")
    if k1 < 0 or k2 < 1 or w > 128:
        raise ValueError(f"re-ranking supports 0 <= k1 <= 127 and 1 <= k2 <= 128 (k1={k1}, k2={k2})")
    if not 1 <= k <= 128:
        raise ValueError(f"re-ranking keeps 1 <= k <= 128 ranks per query (k={k})")
    if not 0.0 <= lambda_value <= 1.0:
        raise ValueError(f"lambda_value must lie in [0, 1] (got {lambda_value})")
    if int(idx_base) != slice_bounds(n, world, rank)[0]:
        raise ValueError(f"sharded_rerank_topk expects rank {rank}'s gallery shard to be its slice_bounds slice "
                         f"(first row {slice_bounds(n, world, rank)[0]}, got idx_base {idx_base})")
    eng = Engine.get(x.device)
    if world == 1:
        y = shard[:n]
    else:
        _, _, per_g = slice_bounds(n, world, rank)
        y = _all_gather_rows(shard[:min(per_g, shard.shape[0])], per_g)[:n]
    X = torch.cat([x, y]).float().contiguous()
    lo, cnt, per = slice_bounds(N, world, rank)
    idx, dd, mx = eng.knn_rowmax(X, w, lo, cnt)
    if world > 1:
        packed = torch.zeros(per, 2 * w + 1, dtype=torch.int32, device=x.device)
        packed[:cnt, :w] = idx.to(torch.int32)
        packed[:cnt, w:2 * w] = dd.view(torch.int32)
        packed[:cnt, 2 * w] = mx.view(torch.int32)
        gathered = torch.empty(world * per, 2 * w + 1, dtype=torch.int32, device=x.device)
        dist.all_gather_into_tensor(gathered, packed)      # rank-major: row r*per + i is global row r*per + i
        if rank != 0:
            return None
        g = gathered[:N]
        idx = g[:, :w].to(torch.int64).contiguous()
        dd = g[:, w:2 * w].contiguous().view(torch.float32)
        mx = g[:, 2 * w].contiguous().view(torch.float32)
    orig = None
    if lambda_value > 0:
        # the first k rows of each query's original ranking can precede the rows without overlap (jac = 1)
        _, orig = eng.l2dist_topk(x.float().contiguous(), y.float().contiguous(), min(k + 8, 128, n))
    return eng.rerank_topk(X, m, idx, dd, mx, k1, k2, lambda_value, k, orig)


def _slice_names(items, world, rank):
    """File names DistributedSliceSampler(items) hands to `rank` (sampler.py:208-219): a contiguous slice of
    ceil(n/world) items whose tail wraps to the head."""
    n = len(items)
    per = int(math.ceil(n * 1.0 / world))
    return [items[(rank * per + i) % n][0] for i in range(per)] if n else []


class Evaluator(object):
    """evaluators.py:170-201.

    Data flow (SURVEY 5 / 8e) when both loaders are given, as examples/test.py does (:127-131): every rank
    keeps the descriptors of its database slice in the HBM that produced them; only the queries are
    all-gathered (6.8k x 16 KiB = 111 MB); every rank ranks all queries against its own slice; the [m,k]
    candidates are all-gathered (8 B each) and merged.  No descriptor is copied to the host and the [m,n]
    distance matrix is never built.  The reference gathers every descriptor to every rank's host RAM
    (:76-101) and computes the dense CPU matrix redundantly on all ranks (:116-130)."""

    _rank_fn = None      # test seam (gloo CPU test): stands in for the CUDA distance/top-k and merge kernels
    _merge_fn = None

    def __init__(self, model):
        self.model = model
        self.rank, _ = _rank_world()
        self.last_stats = {}

    def _resident_inputs(self, query_loader, query, gallery, gallery_loader, vlad, pca, gpu):
        """-> (all queries [m,D] on this GPU, this rank's database rows [per,D], first global row, valid rows)
        or None if a loader did not deliver DistributedSliceSampler slices of `query` / `gallery`."""
        rank, world = _rank_world()
        q_local, q_names = _extract_local(self.model, query_loader, vlad=vlad, pca=pca, gpu=gpu)
        db_local, db_names = _extract_local(self.model, gallery_loader, vlad=vlad, pca=pca, gpu=gpu)
        ok = (q_names == _slice_names(query, world, rank) and db_names == _slice_names(gallery, world, rank))
        if world > 1:
            flag = torch.tensor([1 if ok else 0], device=q_local.device)
            dist.all_reduce(flag, op=dist.ReduceOp.MIN)
            ok = bool(flag.item())
        if not ok:
            return None, (q_local, q_names, db_local, db_names)
        per_q = int(math.ceil(len(query) * 1.0 / world))
        x = _all_gather_rows(q_local, per_q)[: len(query)].contiguous()
        lo, cnt, per = slice_bounds(len(gallery), world, rank)
        self.last_stats = {"d2h_descriptor_bytes": 0,
                           "nvlink_bytes": (world - 1) * per_q * q_local.shape[1] * 4 if world > 1 else 0}
        return (x, db_local, lo, cnt), None

    def evaluate(self, query_loader, dataset, query, gallery, ground_truth, gallery_loader=None,
                 vlad=True, pca=None, rerank=False, gpu=None, sync_gather=False, nms=False, rr_topk=25,
                 lambda_value=0):
        rank, world = _rank_world()
        k = min(10 * (12 if nms else 1), 128)
        resident = None
        if gallery_loader is not None:
            resident, leftovers = self._resident_inputs(query_loader, query, gallery, gallery_loader, vlad, pca, gpu)
        if resident is not None:
            x, shard, lo, cnt = resident
        else:
            # generic loaders (one loader over the union, or a custom sampler): gather by file name
            if gallery_loader is not None:
                q_local, q_names, db_local, db_names = leftovers
                features = self._gather_named(q_local, q_names)
                features.update(self._gather_named(db_local, db_names))
            else:
                local, names = _extract_local(self.model, query_loader, vlad=vlad, pca=pca, gpu=gpu)
                features = self._gather_named(local, names)
            x = torch.stack([features[f] for f, _, _, _ in query])
            lo, cnt, per = slice_bounds(len(gallery), world, rank)
            shard = torch.stack([features[f] for f, _, _, _ in gallery[lo:lo + cnt]]) if cnt else \
                torch.zeros(1, x.shape[1], device=x.device)
        _, idx = sharded_topk(x, shard, k, idx_base=lo, n_valid=cnt, _rank_fn=self._rank_fn, _merge_fn=self._merge_fn)
        if world > 1:
            self.last_stats["nvlink_bytes"] = self.last_stats.get("nvlink_bytes", 0) + (world - 1) * idx.numel() * 8
        recalls = recalls_from_topk(idx.cpu().numpy(), ground_truth, gallery, (1, 5, 10), nms)
        if self.rank == 0:
            print("Recall Scores:")
            for i, kk in enumerate((1, 5, 10)):
                print("  top-{:<4}{:12.1%}".format(kk, recalls[i]))
        if not rerank:
            return recalls
        # evaluators.py:194-201: k-reciprocal re-ranking on sparse data (sharded_rerank_topk): the neighbour pass is
        # split over the ranks, the sparse stage runs on rank 0, and no q-g, q-q or g-g matrix is built.  The other
        # ranks keep the first-pass recalls, as the reference's non-zero ranks score the original matrix.
        if self.rank == 0:
            print("Applying re-ranking ...")
        res = sharded_rerank_topk(x, shard, k, idx_base=lo, n_valid=cnt, k1=rr_topk, k2=1, lambda_value=lambda_value)
        if res is None:
            return recalls
        recalls = recalls_from_topk(res[1].cpu().numpy(), ground_truth, gallery, (1, 5, 10), nms)
        print("Recall Scores:")
        for i, kk in enumerate((1, 5, 10)):
            print("  top-{:<4}{:12.1%}".format(kk, recalls[i]))
        return recalls

    @staticmethod
    def _gather_named(local, names):
        """fname -> GPU row for every image any rank extracted (device all-gather; names travel as objects)."""
        _, world = _rank_world()
        if world == 1:
            return {n: r for n, r in zip(names, local)}
        counts = [None] * world
        dist.all_gather_object(counts, (len(names), names))
        per = max(c for c, _ in counts)
        rows = _all_gather_rows(local, per)
        out = {}
        for r, (c, nm) in enumerate(counts):
            for j in range(c):
                out.setdefault(nm[j], rows[r * per + j])
        return out

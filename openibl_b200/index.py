"""A place index: a geo-tagged gallery extracted once, kept in HBM (sharded as DistributedSliceSampler shards it),
searched many times, saved to disk and loaded again at any world size.

    index = PlaceIndex.build(model, gallery_loader, dataset.db_test, pca=pca)     # collective
    index.save("idx/")                                                            # collective
    index = PlaceIndex.load("idx/", model=model)                                  # collective, any world size
    dist, idx = index.search(descriptors, k=10)                                   # collective
    places = index.localize(images, k=10)      # [[(fname, pid, (x, y), distance), ...] per query]

Each rank keeps its slice_bounds slice of the gallery's fp32 descriptors and their prepared fp16 form
(Engine.prepare_database); a search ranks the queries against every shard (Engine.search_prepared), and the [m,k]
candidates take one packed all-gather and a merge, as in Evaluator.evaluate."""
from __future__ import annotations

import hashlib
import json
import os

import numpy as np
import torch
import torch.distributed as dist

from .engine import Engine
from .evaluators import (_extract_local, _rank_world, _slice_names, extract_cnn_feature, gather_merge_topk,
                         spatial_nms)
from .utils.data.sampler import slice_bounds

__all__ = ["PlaceIndex", "model_fingerprint"]

FORMAT_VERSION = 1


def model_fingerprint(model) -> str:
    """sha256 over the state dict (names with any `module.` prefix stripped, sorted; dtype, shape and bytes)."""
    sd = model.state_dict() if hasattr(model, "state_dict") else model
    h = hashlib.sha256()
    for name in sorted(sd, key=lambda s: s[len("module."):] if s.startswith("module.") else s):
        t = sd[name].detach().cpu().contiguous()
        key = name[len("module."):] if name.startswith("module.") else name
        h.update(f"{key}|{t.dtype}|{tuple(t.shape)}|".encode())
        h.update(t.numpy().tobytes() if t.dtype != torch.bfloat16 else t.view(torch.int16).numpy().tobytes())
    return h.hexdigest()


def _all_ranks_ok(ok: bool, device) -> bool:
    _, world = _rank_world()
    if world == 1:
        return ok
    flag = torch.tensor([1 if ok else 0], device=device)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    return bool(flag.item())


class PlaceIndex:
    # test seam (gloo CPU test): stand-ins for Engine.prepare_database, Engine.search_prepared and the merge kernel
    _prepare_fn = None
    _search_fn = None
    _merge_fn = None

    def __init__(self, gallery, rows, lo, n, dim, vlad=True, pca=None, fingerprint=None, model=None, gpu=None):
        self.gallery = [tuple(it) for it in gallery]
        self.n, self.dim, self.lo = int(n), int(dim), int(lo)
        self.rows = rows                      # this rank's slice_bounds rows [cnt, dim] fp32
        self.vlad, self.pca, self.fingerprint, self.model, self.gpu = vlad, pca, fingerprint, model, gpu
        self._db_ids = [it[1] for it in self.gallery]
        if rows.shape[0] == 0:
            self.prep = None
        elif self._prepare_fn is not None:
            self.prep = type(self)._prepare_fn(rows)
        else:
            self.prep = Engine.get(rows.device).prepare_database(rows)

    # ---- building ------------------------------------------------------------------------------------------------
    @classmethod
    def build(cls, model, loader, gallery, pca=None, vlad=True, gpu=None):
        """Collective: every rank extracts its DistributedSliceSampler slice of `gallery` through `loader` and keeps
        its slice_bounds rows (no wrap-around padding)."""
        rank, world = _rank_world()
        local, names = _extract_local(model, loader, vlad=vlad, pca=pca, gpu=gpu)
        ok = names == _slice_names(gallery, world, rank)
        if not _all_ranks_ok(ok, local.device):
            raise ValueError("PlaceIndex.build: the loader did not deliver this rank's DistributedSliceSampler slice "
                             "of the gallery")
        lo, cnt, _ = slice_bounds(len(gallery), world, rank)
        dim = local.shape[1] if local.numel() else 0
        if world > 1:
            t = torch.tensor([dim], device=local.device)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            dim = int(t.item())
        rows = local[:cnt].float().contiguous() if cnt else torch.empty(0, dim, device=local.device)
        return cls(gallery, rows, lo, len(gallery), dim, vlad, pca, model_fingerprint(model), model, gpu)

    # ---- searching -----------------------------------------------------------------------------------------------
    def search(self, descriptors: torch.Tensor, k: int = 10, nms: bool = False):
        """Collective: every rank passes the same query rows [m, dim].  Returns (dist [m,k], gallery index [m,k]),
        ascending by (distance, index), padded with (inf, -1).  With nms, min(12 k, 128) candidates are ranked and
        the first k distinct places kept (the reference's spatial_nms, evaluators.py:132-140)."""
        q = descriptors.float().contiguous()
        m, d = q.shape
        _, world = _rank_world()
        shape_ok = d == self.dim
        if world > 1:
            shp = torch.tensor([m, d], dtype=torch.int64, device=q.device)
            allshp = torch.empty(world * 2, dtype=torch.int64, device=q.device)
            dist.all_gather_into_tensor(allshp, shp)
            shape_ok = shape_ok and bool((allshp.view(world, 2) == shp).all())
        if not shape_ok:
            raise ValueError(f"PlaceIndex.search: every rank must pass the same [m, {self.dim}] query rows "
                             f"(this rank: [{m}, {d}])")
        if not 1 <= k <= 128:
            raise ValueError(f"PlaceIndex.search keeps 1 <= k <= 128 ranks (k={k})")
        kk = min(12 * k, 128) if nms else k
        if self.prep is None:
            cd = torch.full((m, kk), float("inf"), device=q.device)
            ci = torch.full((m, kk), -1, dtype=torch.int64, device=q.device)
        elif self._search_fn is not None:
            cd, ci = type(self)._search_fn(q, self.prep, kk, self.lo)
        else:
            cd, ci = Engine.get(q.device).search_prepared(q, self.prep, kk, idx_base=self.lo)
        merge = type(self)._merge_fn if self._merge_fn is not None else Engine.get(q.device).topk_merge
        cd, ci = gather_merge_topk(cd, ci, kk, merge)
        if not nms:
            return cd, ci
        od = torch.full((m, k), float("inf"))
        oi = torch.full((m, k), -1, dtype=torch.int64)
        cdh, cih = cd.cpu(), ci.cpu().numpy()
        for r in range(m):
            pred = cih[r][cih[r] >= 0]
            pos = {p: j for j, p in reversed(list(enumerate(pred)))}
            kept = spatial_nms(list(pred), self._db_ids, kk)[:k]
            for j, p in enumerate(kept):
                oi[r, j] = int(p)
                od[r, j] = cdh[r, pos[p]]
        return od.to(cd.device), oi.to(ci.device)

    def localize(self, images, k: int = 10):
        """Collective: extracts the image batch on the calling rank (with the index's PCA), searches, and returns
        per query the top-k [(fname, pid, (x, y), distance), ...]."""
        if self.model is None:
            raise ValueError("PlaceIndex.localize needs the model: build the index, or load it with model=...")
        with torch.no_grad():
            x = extract_cnn_feature(self.model, images, self.vlad, gpu=self.gpu)
            if self.pca is not None:
                if self.pca.weight is None:
                    self.pca.load(gpu=self.gpu)
                x = self.pca.infer(x)
        dd, ii = self.search(x, k)
        dd, ii = dd.cpu().tolist(), ii.cpu().tolist()
        out = []
        for dr, ir in zip(dd, ii):
            out.append([(self.gallery[i][0], self.gallery[i][1], (self.gallery[i][2], self.gallery[i][3]), dv)
                        for dv, i in zip(dr, ir) if i >= 0])
        return out

    # ---- persistence ---------------------------------------------------------------------------------------------
    def save(self, path: str):
        """Collective: rank r writes rows_<r>.npy (its fp32 slice); rank 0 writes index.json (and the PCA
        parameters, pca_params.npz, when the index was built with PCA).  The fp16 plane is not stored."""
        rank, world = _rank_world()
        os.makedirs(path, exist_ok=True)
        np.save(os.path.join(path, f"rows_{rank}.npy"), self.rows.detach().cpu().numpy().astype(np.float32))
        if rank == 0:
            shards = []
            for r in range(world):
                lo, cnt, _ = slice_bounds(self.n, world, r)
                shards.append({"file": f"rows_{r}.npy", "first": lo, "count": cnt})
            meta = {"format_version": FORMAT_VERSION, "n": self.n, "dim": self.dim, "vlad": bool(self.vlad),
                    "model_sha256": self.fingerprint, "gallery": [list(it) for it in self.gallery],
                    "shards": shards, "pca": None}
            if self.pca is not None:
                np.savez(os.path.join(path, "pca_params.npz"), **self.pca._read())
                open(os.path.join(path, "pca_params"), "wb").close()   # PCA reads <path>.npz behind an empty marker
                meta["pca"] = {"n_components": int(self.pca.pca_n_components),
                               "whitening": bool(self.pca.pca_whitening), "file": "pca_params.npz"}
            tmp = os.path.join(path, "index.json.tmp")
            with open(tmp, "w") as f:
                json.dump(meta, f)
            os.replace(tmp, os.path.join(path, "index.json"))
        if world > 1:
            dist.barrier()

    @classmethod
    def load(cls, path: str, gpu=None, model=None, device=None):
        """Collective, at any world size: each rank memory-maps the row files that overlap its slice_bounds slice,
        copies the slice to its GPU and prepares it.  With `model`, its fingerprint must match the saved one."""
        rank, world = _rank_world()
        with open(os.path.join(path, "index.json")) as f:
            meta = json.load(f)
        if meta.get("format_version") != FORMAT_VERSION:
            raise ValueError(f"{path}/index.json: format version {meta.get('format_version')}, "
                             f"this code reads {FORMAT_VERSION}")
        if model is not None and model_fingerprint(model) != meta["model_sha256"]:
            raise ValueError(f"{path}: the index was built with a different model (state-dict sha256 "
                             f"{meta['model_sha256'][:12]}…, this model {model_fingerprint(model)[:12]}…)")
        n, dim = int(meta["n"]), int(meta["dim"])
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device() if gpu is None else gpu)
        lo, cnt, _ = slice_bounds(n, world, rank)
        rows = torch.empty(cnt, dim, device=device)
        for sh in meta["shards"]:
            a, b = max(lo, sh["first"]), min(lo + cnt, sh["first"] + sh["count"])
            if a >= b:
                continue
            fp = os.path.join(path, sh["file"])
            if not os.path.isfile(fp):
                raise FileNotFoundError(f"{fp}: missing shard file of the place index (rows {sh['first']}.."
                                        f"{sh['first'] + sh['count'] - 1})")
            arr = np.load(fp, mmap_mode="r")
            if arr.ndim != 2 or arr.shape[1] != dim or arr.shape[0] != sh["count"]:
                raise ValueError(f"{fp}: shape {arr.shape}, index.json says [{sh['count']}, {dim}]")
            rows[a - lo:b - lo] = torch.from_numpy(np.array(arr[a - sh["first"]:b - sh["first"]], dtype=np.float32))
        pca = None
        if meta.get("pca"):
            from .pca import PCA
            p = meta["pca"]
            base = os.path.join(path, p["file"][: -len(".npz")])
            for fp in (base, base + ".npz"):
                if not os.path.isfile(fp):
                    raise FileNotFoundError(f"{fp}: missing PCA parameters of the place index")
            pca = PCA(p["n_components"], p["whitening"], base)
        return cls([tuple(it) for it in meta["gallery"]], rows, lo, n, dim, meta["vlad"], pca,
                   meta["model_sha256"], model, gpu)

"""DistributedSliceSampler (ibl/utils/data/sampler.py:194-223): rank r reads the r-th contiguous
slice of ceil(N/world) items, the tail wrapping to the head; extract_features un-pads by
truncation.  Part of the hot-path contract (SURVEY 8e).

Like the reference module (sampler.py:9-12) this one re-exports torch's samplers, so that
`from ibl.utils.data.sampler import SubsetRandomSampler` (examples/cluster.py:21) resolves."""
import math

import torch.distributed as dist
from torch.utils.data import BatchSampler  # noqa: F401
from torch.utils.data.sampler import (  # noqa: F401
    RandomSampler, Sampler, SequentialSampler, SubsetRandomSampler, WeightedRandomSampler)


def slice_bounds(n, world, rank):
    """(first, count, padded_count) of rank's slice."""
    per = int(math.ceil(n * 1.0 / world))
    lo = min(rank * per, n)
    return lo, max(0, min(n, lo + per) - lo), per


class DistributedSliceSampler(Sampler):
    def __init__(self, dataset, num_replicas=None, rank=None):
        if num_replicas is None:
            if not dist.is_available():
                raise RuntimeError("Requires distributed package to be available")
            num_replicas = dist.get_world_size()
        if rank is None:
            if not dist.is_available():
                raise RuntimeError("Requires distributed package to be available")
            rank = dist.get_rank()
        self.dataset, self.num_replicas, self.rank = dataset, num_replicas, rank
        n = len(dataset)
        self.num_samples = int(math.ceil(n * 1.0 / num_replicas))
        self.total_size = self.num_samples * num_replicas

    def __iter__(self):
        n = len(self.dataset)
        start = self.rank * self.num_samples
        return iter([(start + i) % n if start + i >= n else start + i for i in range(self.num_samples)])

    def __len__(self):
        return self.num_samples


# ---------------------------------------------------------------------------------------------------------------
# Training tuple samplers (reference ibl/utils/data/sampler.py:15-192).  The expensive part of their refresh -- a full
# argsort of the [queries, gallery] distance matrix, torch.argsort on the CPU in the reference (:49, :129) -- runs on
# the device (ibl_argsort_rows); tuple assembly (easiest positive, random negative pool + cached hard negatives,
# Jaccard-ranked difficult positives) is host logic with the same `random` calls, so that with the same RNG state
# and the same ranking the yielded tuples are identical to the reference's.
# ---------------------------------------------------------------------------------------------------------------
import random

import torch


def _argsort_rows_on_device(distmat):
    """[m,n] distances (CPU or CUDA tensor / ndarray) -> CPU LongTensor [m,n], sorted by (distance, index)."""
    from ...engine import Engine
    d = torch.as_tensor(distmat).float()
    eng = Engine.get(d.device if d.is_cuda else None)
    dev = torch.device("cuda", eng.device)
    out = torch.empty(d.shape, dtype=torch.int64)
    rows = max(1, (1 << 27) // max(d.shape[1], 1))            # bound the device copy of a CPU matrix to 512 MB chunks
    for r0 in range(0, d.shape[0], rows):
        out[r0:r0 + rows] = eng.argsort_rows(d[r0:r0 + rows].to(dev).contiguous()).cpu()
    return out


class _TupleSamplerBase(Sampler):
    def __init__(self, query_source, gallery_source, pos_list, neg_list, neg_num, neg_pool, sub_length, num_replicas, rank):
        if num_replicas is None:
            if not dist.is_available():
                raise RuntimeError("Requires distributed package to be available")
            num_replicas = dist.get_world_size()
        if rank is None:
            if not dist.is_available():
                raise RuntimeError("Requires distributed package to be available")
            rank = dist.get_rank()
        self.num_replicas, self.rank, self.epoch = num_replicas, rank, 0
        self.query_source, self.gallery_source = query_source, gallery_source
        self.pos_list, self.neg_list = pos_list, neg_list
        self.neg_num, self.neg_pool = neg_num, neg_pool
        self.sub_set = list(range(len(query_source)))
        self.sub_length = sub_length
        if self.sub_length is None:
            self.sub_length = len(query_source)
            self._resize()
        self.sort_idx = None
        self.neg_cache = [[]] * len(query_source)

    def _resize(self):
        self.sub_length_dist = int(math.ceil(self.sub_length * 1.0 / self.num_replicas))
        self.total_size = self.sub_length_dist * self.num_replicas

    def _set_ranking(self, distmat, sub_set):
        assert distmat.shape[0] == len(self.query_source) and distmat.shape[1] == len(self.gallery_source)
        self.sort_idx = _argsort_rows_on_device(distmat)
        self.sub_set = sub_set
        self.sub_length = len(sub_set)
        self._resize()

    def __len__(self):
        return self.sub_length_dist

    def set_epoch(self, epoch):
        self.epoch = epoch

    def _my_anchors(self):
        order = list(range(self.sub_length))
        order += order[: self.total_size - len(order)]          # pad to a multiple of the world size
        assert len(order) == self.total_size
        mine = order[self.rank:self.total_size:self.num_replicas]
        assert len(mine) == self.sub_length_dist
        return [self.sub_set[i] for i in mine]

    def _ranked_positives(self, anchor):
        pos = set(self.pos_list[anchor])
        return [g for g in self.sort_idx[anchor].tolist() if g in pos]

    def _hard_negatives(self, anchor):
        """sampler.py:78-85: a random pool of candidate RANKS (gallery minus the potential positives) united with the
        ranks of last epoch's negatives; the neg_num best-ranked of them."""
        banned = set(self.neg_list[anchor])
        cand = [g for g in self.sort_idx[anchor].tolist() if g not in banned]
        pool = random.sample(range(len(cand)), min(self.neg_pool, len(cand)))
        rank_of = {g: i for i, g in enumerate(cand)}
        cached = [rank_of[g] for g in self.neg_cache[anchor]]
        ranks = sorted(set(pool) | set(cached))[: self.neg_num]
        chosen = [cand[i] for i in ranks]
        self.neg_cache[anchor] = chosen
        assert len(chosen) == self.neg_num
        return chosen


class DistributedRandomTupleSampler(_TupleSamplerBase):
    """sampler.py:15-89: (anchor, easiest positive, neg_num hardest pooled negatives); gallery ids are offset by
    len(query_source) because the training set concatenates queries and gallery."""

    def __init__(self, query_source, gallery_source, pos_list, neg_list, neg_num=10, neg_pool=1000, sub_length=None,
                 num_replicas=None, rank=None):
        super().__init__(query_source, gallery_source, pos_list, neg_list, neg_num, neg_pool, sub_length, num_replicas, rank)

    def sort_gallery(self, distmat, sub_set):
        self._set_ranking(distmat, sub_set)

    def __iter__(self):
        off = len(self.query_source)
        for anchor in self._my_anchors():
            pos = self._ranked_positives(anchor)[0]
            negs = self._hard_negatives(anchor)
            yield [anchor, pos + off] + [n + off for n in negs]


class DistributedRandomDiffTupleSampler(_TupleSamplerBase):
    """sampler.py:92-192 (SFRS): additionally pos_num "difficult" positives -- among the pos_pool best-ranked true
    positives, those that the k-reciprocal (Jaccard) distance ranks no later than the original distance does, in the
    order sampler.py:158-171 defines."""

    def __init__(self, query_source, gallery_source, pos_list, neg_list, pos_num=10, pos_pool=20, neg_num=10,
                 neg_pool=1000, sub_length=None, num_replicas=None, rank=None):
        super().__init__(query_source, gallery_source, pos_list, neg_list, neg_num, neg_pool, sub_length, num_replicas, rank)
        self.pos_num, self.pos_pool = pos_num, pos_pool
        self.distmat_jac = None

    def sort_gallery(self, distmat, distmat_jac, sub_set):
        self._set_ranking(distmat, sub_set)
        self.distmat_jac = distmat_jac

    def _difficult_positives(self, anchor, ranked_pos):
        pool = ranked_pos[: self.pos_pool]
        jac = torch.as_tensor(self.distmat_jac[anchor])[torch.tensor(pool, dtype=torch.long)]
        by_jac = torch.argsort(jac, dim=0)                     # by_jac[r] = pool position with the r-th smallest Jaccard distance
        n = by_jac.numel()
        gap = torch.arange(n) - by_jac                         # r - pool position
        slots = torch.arange(n)
        moved = slots[gap < 0]                                 # Jaccard ranks where a LATER pool entry moved forward
        moved = moved[torch.argsort(gap[gap < 0], dim=0)]      # largest jump first
        keep = torch.cat((moved, slots[gap == 0]), dim=0)[: self.pos_num]
        return torch.tensor(pool, dtype=torch.long)[by_jac[keep]].tolist()

    def __iter__(self):
        off = len(self.query_source)
        for anchor in self._my_anchors():
            ranked = self._ranked_positives(anchor)
            diff = self._difficult_positives(anchor, ranked)
            negs = self._hard_negatives(anchor)
            yield [anchor, ranked[0] + off] + [n + off for n in negs] + [p + off for p in diff]

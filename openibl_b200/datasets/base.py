"""Place-recognition split loader: the attribute contract of the reference's ibl/utils/data/dataset.py:49-121
(q_train / db_train / train / q_val / db_val / q_test / db_test lists of (fname, pid, utm_x, utm_y), the
*_pos / *_neg ground-truth lists, images_dir) read from the `meta[_scale].json` + `splits[_scale].json` pair
the reference's `arrange()` writes.  Host-side glue: nothing here is on the accelerated path."""
from __future__ import annotations

import os.path as osp

import numpy as np
# imported with the package, as the reference's dataset module does: importing scikit-learn draws from the global
# `random`, and a script that seeds `random` before creating a dataset must see the reference's stream afterwards
from sklearn.neighbors import NearestNeighbors

from ..utils.serialization import read_json


def items_of(identities, utm, pids):
    """(fname, pid, x, y) for every image of every place id, sorted (dataset.py:11-21, relabel=False)."""
    out = [(fname, pid, utm[pid][0], utm[pid][1]) for pid in pids for fname in identities[pid]]
    return sorted(out)


def radius_groundtruth(query, gallery, pos_radius, neg_radius=None):
    """dataset.py:23-42: for every query the gallery indices within `pos_radius` metres (UTM) that belong to a
    different place id; queries without any are dropped (their indices are returned as `kept`).  With
    `neg_radius`, also the indices within that radius (the "not a negative" set)."""
    nn = NearestNeighbors(n_jobs=-1).fit(np.asarray([[g[2], g[3]] for g in gallery], dtype=np.float64))
    q_xy = np.asarray([[q[2], q[3]] for q in query], dtype=np.float64)
    _, near = nn.radius_neighbors(q_xy, radius=pos_radius)
    pos, kept = [], []
    for qi, cand in enumerate(near):
        mine = [int(g) for g in cand.tolist() if gallery[g][1] != query[qi][1]]
        if mine:
            pos.append(mine)
            kept.append(qi)
    if neg_radius is None:
        return pos, kept
    _, wide = nn.radius_neighbors(q_xy, radius=neg_radius)
    return pos, [w.tolist() for w in wide], kept


class PlaceDataset(object):
    intra_thres, inter_thres = 10, 25       # metres: training positives / potential-positive radius

    def __init__(self, root):
        self.root = root
        self.train, self.q_val, self.db_val, self.q_test, self.db_test = [], [], [], [], []
        self.train_pos, self.train_neg, self.val_pos, self.val_neg, self.test_pos, self.test_neg = [], [], [], [], [], []

    @property
    def images_dir(self):
        return osp.join(self.root, "raw")

    def _json_paths(self, scale=None):
        tag = "" if scale is None else "_" + scale
        return osp.join(self.root, "meta%s.json" % tag), osp.join(self.root, "splits%s.json" % tag)

    def _check_integrity(self, scale=None):
        return all(osp.isfile(p) for p in self._json_paths(scale))

    def load(self, verbose, scale=None):
        meta_p, splits_p = self._json_paths(scale)
        meta, splits = read_json(meta_p), read_json(splits_p)
        ident, utm = meta["identities"], meta["utm"]
        part = {k: items_of(ident, utm, sorted(splits[k])) for k in ("q_train", "db_train", "q_val", "db_val", "q_test", "db_test")}
        self.q_train, self.db_train = part["q_train"], part["db_train"]
        self.train = self.q_train + self.db_train
        self.q_val, self.db_val, self.q_test, self.db_test = part["q_val"], part["db_val"], part["q_test"], part["db_test"]
        self.train_pos, neg, kept = radius_groundtruth(self.q_train, self.db_train, self.intra_thres, self.inter_thres)
        self.train_neg = [neg[i] for i in kept]
        self.q_train = [self.q_train[i] for i in kept]
        self.val_pos, kept = radius_groundtruth(self.q_val, self.db_val, 25)
        assert len(kept) == len(self.q_val), "every validation query needs a positive within 25 m"
        self.test_pos, kept = radius_groundtruth(self.q_test, self.db_test, 25)
        assert len(kept) == len(self.q_test), "every test query needs a positive within 25 m"
        if verbose and _rank() == 0:
            print(self.__class__.__name__, "dataset loaded")
            print("  subset        | # pids | # images")
            print("  ---------------------------------")
            for label, items in (("train_query", self.q_train), ("train_gallery", self.db_train), ("val_query", self.q_val),
                                 ("val_gallery", self.db_val), ("test_query", self.q_test), ("test_gallery", self.db_test)):
                print("  {:<13} | {:5d}  | {:8d}".format(label, len({it[1] for it in items}), len(items)))


def _rank():
    try:
        import torch.distributed as dist
        return dist.get_rank()
    except Exception:
        return 0

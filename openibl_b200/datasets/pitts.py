"""Pittsburgh 30k / 250k (reference ibl/datasets/pitts.py:11-103): `<root>/raw/pitts<scale>_{train,val,test}.mat`
(NetVLAD's dbStruct) -> `meta_<scale>.json` + `splits_<scale>.json`, then the common split loader."""
from __future__ import annotations

import os.path as osp

from ..utils.dist_utils import synchronize
from ..utils.serialization import read_mat, write_json
from .base import PlaceDataset, _rank


def read_dbstruct(path, time_stamp=False):
    """dbStruct fields used: [1] dbImage, [2] utmDb (2 x n), [3] qImage, [4] utmQ (2 x n) (pitts.py:11-23).  With
    `time_stamp` (Tokyo Time Machine), a time-stamp vector follows each UTM matrix, so qImage / utmQ sit at [4] / [5]
    (tokyo.py:12-23)."""
    s = read_mat(path)
    names = lambda cell: [c[0].item() for c in cell]
    ts = int(time_stamp)
    return {"db": names(s[1]), "db_utm": s[2].T, "q": names(s[3 + ts]), "q_utm": s[4 + ts].T}


class Pittsburgh(PlaceDataset):
    def __init__(self, root, scale="250k", verbose=True):
        super().__init__(root)
        self.scale = scale
        self.arrange()
        self.load(verbose, scale)

    def arrange(self):
        if self._check_integrity(self.scale):
            return
        raw = osp.join(self.root, "raw")
        if not osp.isdir(raw):
            raise RuntimeError("Dataset not found.")
        identities, utms = [], []
        place_of = {"q": {}, "db": {}}                 # panorama id ('000123') -> place id, per role
        sub_dir = {"q": osp.join("Pittsburgh", "queries"), "db": osp.join("Pittsburgh", "images")}
        splits = {}
        for split in ("train", "val", "test"):
            s = read_dbstruct(osp.join(raw, "pitts%s_%s.mat" % (self.scale, split)))
            for role in ("q", "db"):
                fresh = []
                for fpath, utm in zip(s[role], s[role + "_utm"]):
                    key = fpath.split("_")[0]
                    pid = place_of[role].get(key)
                    if pid is None:
                        pid = place_of[role][key] = len(identities)
                        identities.append([])
                        utms.append(utm.tolist())
                        fresh.append(pid)
                    assert utms[pid] == utm.tolist(), "one panorama, one UTM position"
                    identities[pid].append(osp.join(sub_dir[role], fpath))
                splits["%s_%s" % (role, split)] = sorted(fresh)
        meta_p, splits_p = self._json_paths(self.scale)
        if _rank() == 0:
            write_json({"name": "Pittsburgh_" + self.scale, "identities": identities, "utm": utms}, meta_p)
            write_json(splits, splits_p)
        synchronize()

"""Tokyo 24/7 + Tokyo Time Machine (reference ibl/datasets/tokyo.py:12-157): `<root>/raw/tokyoTM_{train,val}.mat` and
`<root>/raw/tokyo247.mat` (NetVLAD's dbStruct) -> `meta.json` + `splits.json`, then the common split loader.

Time Machine images are grouped into places (path component [1]) and, within a place, into one identity per time stamp
(component [2]).  Training places keep every time stamp as a training identity; every validation place with more than
one time stamp gives one of them, drawn with `random.randrange` on the global `random` module, as its query identity.
Tokyo 24/7 is the test split: queries that share a UTM position form one place, database images one place per
directory, named .png as the released database is.  For the same tree and the same `random` state the two json files
are byte-identical to the reference's, and the same number of values is drawn from `random`."""
from __future__ import annotations

import os.path as osp
import random

import numpy as np

from ..utils.dist_utils import synchronize
from ..utils.serialization import write_json
from .base import PlaceDataset, _rank
from .pitts import read_dbstruct

TM_ROOT = osp.join("tokyoTM", "images")
DB_ROOT = osp.join("tokyo247", "images")
Q_ROOT = osp.join("tokyo247", "query")


class Tokyo(PlaceDataset):
    def __init__(self, root, scale=None, verbose=True):
        super().__init__(root)
        self.arrange()
        self.load(verbose)

    def arrange(self):
        # every rank looks before rank 0 writes, so that all ranks take the same branch (and draw the same values
        # from `random`) however their start-up times differ
        present = self._check_integrity()
        synchronize()
        if present:
            return
        raw = osp.join(self.root, "raw")
        if not osp.isdir(raw):
            raise RuntimeError("Dataset not found.")
        identities, utms = [], []             # per Time Machine place: one list of paths per time stamp
        place_of, ts_of, seen = {}, [], []    # place name -> pid; per pid: time stamp -> slot, set of paths

        def register_tm(split):
            s = read_dbstruct(osp.join(raw, "tokyoTM_%s.mat" % split), time_stamp=True)
            fresh = []
            for fpath, utm in zip(s["q"] + s["db"], np.concatenate((s["q_utm"], s["db_utm"]))):
                parts = fpath.split("/")
                pid = place_of.get(parts[1])
                if pid is None:
                    pid = place_of[parts[1]] = len(identities)
                    identities.append([])
                    utms.append(utm.tolist())
                    ts_of.append({})
                    seen.append(set())
                    fresh.append(pid)
                slot = ts_of[pid].get(parts[2])
                if slot is None:
                    slot = ts_of[pid][parts[2]] = len(identities[pid])
                    identities[pid].append([])
                path = osp.join(TM_ROOT, fpath)
                if path not in seen[pid]:
                    seen[pid].add(path)
                    identities[pid][slot].append(path)
                assert utms[pid] == utm.tolist(), "one place, one UTM position"
            return set(fresh)

        train_pids = register_tm("train")
        val_pids = register_tm("val")

        new_identities, new_utms = [], []
        q_train, q_val, db_val = [], [], []

        def add(group, pid, paths):
            group.append(len(new_identities))
            new_identities.append(sorted(paths))
            new_utms.append(utms[pid])

        for pid, per_ts in enumerate(identities):
            if pid in train_pids:
                for paths in per_ts:
                    add(q_train, pid, paths)
            if pid in val_pids:
                if len(per_ts) > 1:
                    add(q_val, pid, per_ts.pop(random.randrange(len(per_ts))))
                for paths in per_ts:
                    add(db_val, pid, paths)
        identities, utms = new_identities, new_utms

        s = read_dbstruct(osp.join(raw, "tokyo247.mat"), time_stamp=False)
        q_test, db_test = [], []
        for role, group, key_of, name_of, sub_dir in (
                ("q", q_test, lambda f, u: str(u[0]) + "_" + str(u[1]), lambda f: f, Q_ROOT),
                ("db", db_test, lambda f, u: osp.dirname(f), lambda f: f[:-3] + "png", DB_ROOT)):
            place = {}
            for fpath, utm in zip(s[role], s[role + "_utm"]):
                key = key_of(fpath, utm)
                pid = place.get(key)
                if pid is None:
                    pid = place[key] = len(identities)
                    identities.append([])
                    utms.append(utm.tolist())
                    group.append(pid)
                identities[pid].append(osp.join(sub_dir, name_of(fpath)))
                assert utms[pid] == utm.tolist(), "one place, one UTM position"

        splits = {"q_train": sorted(q_train), "db_train": sorted(q_train), "q_val": sorted(q_val),
                  "db_val": sorted(db_val), "q_test": sorted(q_test), "db_test": sorted(db_test)}
        meta_p, splits_p = self._json_paths()
        if _rank() == 0:
            write_json({"name": "Tokyo", "identities": identities, "utm": utms}, meta_p)
            write_json(splits, splits_p)
        synchronize()

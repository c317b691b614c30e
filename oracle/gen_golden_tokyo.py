#!/usr/bin/env python
"""Golden vectors for the Tokyo arrangement: the UNMODIFIED reference `ibl.datasets.create('tokyo', root)`
(ibl/datasets/tokyo.py:25-157) on the seeded synthetic tree of `write_synthetic_tokyo_tree`, with the global `random`
seeded first, as the training drivers seed it.  Stored: the bytes of meta.json and splits.json, the loaded split lists
and *_pos lists, and the `random.random()` drawn right after the arrangement (it shows how many values the
arrangement took).  TEST INFRASTRUCTURE; build container only (needs /root/reference).

    python oracle/gen_golden_tokyo.py      # writes tests/golden/tokyo_arrange.npz
"""
import os, random, sys, tempfile, types, warnings
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.gen_golden_trainer import write_npz
from openibl_b200.datasets.synthetic import write_synthetic_tokyo_tree
sys.modules.setdefault("h5py", types.ModuleType("h5py"))
sys.path.insert(0, os.environ.get("IBL_REFERENCE", "/root/reference"))
warnings.filterwarnings("ignore")
from ibl import datasets                      # the reference's

TREE_SEED, RANDOM_SEED = 5, 43
SPLITS = ("q_train", "db_train", "q_val", "db_val", "q_test", "db_test")


def ragged(lists):
    return np.asarray([len(x) for x in lists], dtype=np.int64), np.asarray([int(i) for x in lists for i in x], dtype=np.int64)


if __name__ == "__main__":
    assert datasets.__file__.startswith(os.path.abspath(os.environ.get("IBL_REFERENCE", "/root/reference")))
    with tempfile.TemporaryDirectory() as tmp:
        root = write_synthetic_tokyo_tree(os.path.join(tmp, "tokyo"), seed=TREE_SEED)
        random.seed(RANDOM_SEED)
        ds = datasets.create("tokyo", root, verbose=False)
        out = {"tree_seed": np.int64(TREE_SEED), "random_seed": np.int64(RANDOM_SEED),
               "next_random": np.float64(random.random())}
        for name in ("meta.json", "splits.json"):
            out[name.replace(".", "_")] = np.frombuffer(open(os.path.join(root, name), "rb").read(), dtype=np.uint8)
        for split in SPLITS:
            items = getattr(ds, split)
            out[split + "_fname"] = np.asarray([it[0] for it in items], dtype=str)
            out[split + "_pid"] = np.asarray([it[1] for it in items], dtype=np.int64)
            out[split + "_utm"] = np.asarray([[it[2], it[3]] for it in items], dtype=np.float64).reshape(-1, 2)
        for k in ("train_pos", "val_pos", "test_pos"):
            out[k + "_len"], out[k + "_flat"] = ragged(getattr(ds, k))
    path = os.path.join(ROOT, "tests", "golden", "tokyo_arrange.npz")
    write_npz(path, out)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB; splits",
          {s: len(out[s + "_pid"]) for s in SPLITS}, "next random", float(out["next_random"]))

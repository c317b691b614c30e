"""Tokyo 24/7 (+ Time Machine) -- reference ibl/datasets/tokyo.py:12-157.  The split loader reads the
`meta.json` / `splits.json` pair that the reference's `arrange()` writes; arranging from the raw .mat files
(time-machine regrouping with a random validation query per place, tokyo.py:41-95) is not ported -- run the
reference's `ibl.datasets.create('tokyo', root)` once to produce the two json files."""
from __future__ import annotations

import os.path as osp

from .base import PlaceDataset


class Tokyo(PlaceDataset):
    def __init__(self, root, scale=None, verbose=True):
        super().__init__(root)
        if not self._check_integrity():
            if not osp.isdir(osp.join(root, "raw")):
                raise RuntimeError("Dataset not found.")
            raise NotImplementedError(
                "Tokyo 24/7: meta.json / splits.json are missing under %r; arranging them from the raw .mat files "
                "is host-side dataset preparation outside the GPU hot path -- produce them once with the "
                "reference's ibl.datasets.create('tokyo', root)" % root)
        self.load(verbose)

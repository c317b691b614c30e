"""`ibl` -- the reference's package name, served by the H100 (sm_90a) engine.

A thin alias layer so that code written against yxgeee/OpenIBL (`from ibl import models`,
`from ibl.evaluators import Evaluator, extract_features, pairwise_distance`, `from ibl.pca import PCA`,
`from ibl.utils.data.sampler import DistributedSliceSampler`, ...; examples/test.py:17-26) imports
the H100-native host mirror in openibl_b200/ unchanged."""
import sys as _sys

import openibl_b200 as _pkg
from openibl_b200 import datasets, evaluators, index, models, pca, trainers, utils  # noqa: F401
from openibl_b200.utils import data as _data, dist_utils as _du, logging as _lg, meters as _mt, rerank as _rr, serialization as _sr
from openibl_b200.utils.data import preprocessor as _pp, sampler as _sm

for _name, _mod in {
    "models": models, "evaluators": evaluators, "index": index, "pca": pca, "trainers": trainers, "utils": utils, "datasets": datasets,
    "utils.data": _data, "utils.dist_utils": _du, "utils.logging": _lg, "utils.meters": _mt,
    "utils.serialization": _sr, "utils.rerank": _rr, "utils.data.preprocessor": _pp, "utils.data.sampler": _sm,
}.items():
    _sys.modules["ibl." + _name] = _mod

__version__ = "0.0.1+b200"

#!/usr/bin/env python
"""End-to-end evaluation through the reference-shaped API on a synthetic place-recognition set.

Same flow as the reference's examples/test.py (main_worker, :77-133) -- init_dist, build loaders with
DistributedSliceSampler, models.create('vgg16') + 'netvlad' + 'embednet', DistributedDataParallel,
Evaluator(model).evaluate(...) -- but the images are generated from seeds instead of being read from the
Pittsburgh / Tokyo files (no datasets on the build or GPU boxes).  Every query is a noisy copy of one
database image, so Recall@1 is high but not trivially 100 %.

    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 examples/eval_synthetic.py \
        --launcher pytorch --n-db 96 --n-q 24 --height 128 --width 160
"""
from __future__ import print_function, absolute_import

import argparse
import os
import os.path as osp
import sys

import numpy as np
import torch
from torch import nn
from torch.utils.data import DataLoader, Dataset

sys.path.insert(0, osp.dirname(osp.dirname(osp.abspath(__file__))))

from ibl import datasets, models  # noqa: E402
from ibl.evaluators import Evaluator  # noqa: E402
from ibl.pca import PCA  # noqa: E402
from ibl.utils.data.sampler import DistributedSliceSampler  # noqa: E402
from ibl.utils.dist_utils import init_dist, synchronize  # noqa: E402


class SeededImages(Dataset):
    """(img, fname, pid, x, y) like ibl.utils.data.preprocessor.Preprocessor, images from seeds."""

    def __init__(self, items, height, width, noise=0.35):
        self.items, self.h, self.w, self.noise = items, height, width, noise

    def __len__(self):
        return len(self.items)

    def __getitem__(self, index):
        fname, pid, x, y = self.items[index]
        base = int(x)                                     # database image this one is derived from
        g = torch.Generator().manual_seed(1000 + base)
        img = torch.randn(3, self.h, self.w, generator=g)
        if fname.startswith("q/"):
            gq = torch.Generator().manual_seed(500000 + pid)
            img = img + self.noise * torch.randn(3, self.h, self.w, generator=gq)
        return img, fname, pid, x, y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launcher", default="pytorch", choices=["pytorch", "slurm"])
    ap.add_argument("--tcp-port", default="5017")
    ap.add_argument("--n-db", type=int, default=96)
    ap.add_argument("--n-q", type=int, default=24)
    ap.add_argument("--height", type=int, default=128)
    ap.add_argument("--width", type=int, default=160)
    ap.add_argument("--test-batch-size", type=int, default=8)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--expect-recalls", default="", help="comma-separated recalls to assert (tests)")
    ap.add_argument("--rerank", action="store_true", help="k-reciprocal re-ranking, as examples/test.py --rerank")
    ap.add_argument("--rr-topk", type=int, default=25)
    ap.add_argument("--lambda-value", type=float, default=0.0)
    ap.add_argument("--nms", action="store_true", help="spatial NMS on the ranking, as examples/test.py --nms")
    args = ap.parse_args()

    init_dist(args.launcher, args)                        # one process per GPU, NCCL
    synchronize()
    ds = datasets.create("synthetic", None, n_db=args.n_db, n_q=args.n_q, seed=args.seed)

    def loader(items):
        return DataLoader(SeededImages(items, args.height, args.width), batch_size=args.test_batch_size,
                          num_workers=0, sampler=DistributedSliceSampler(items), shuffle=False, pin_memory=True)

    torch.manual_seed(args.seed)                          # identical random-init weights on every rank
    base_model = models.create("vgg16", pretrained=False)
    pool_layer = models.create("netvlad", dim=base_model.feature_dim)
    # _init_params-style NetVLAD parameters (unit-norm centroids, alpha ~ 280): with the default
    # random init every descriptor is dominated by the centroid term and all distances are ~1e-6
    from openibl_b200 import synth
    p = synth.make_netvlad_params(seed=args.seed, sharp=True)
    pool_layer.centroids.data.copy_(p["centroids"])
    pool_layer.conv.weight.data.copy_(p["conv_weight"])
    model = models.create("embednet", base_model, pool_layer)
    model.cuda(args.gpu)
    model = nn.parallel.DistributedDataParallel(model, device_ids=[args.gpu], output_device=args.gpu,
                                                find_unused_parameters=True)
    evaluator = Evaluator(model)
    dataset = sorted(list(set(ds.q_test) | set(ds.db_test)))
    recalls = evaluator.evaluate(loader(ds.q_test), dataset, ds.q_test, ds.db_test, ds.test_pos,
                                 gallery_loader=loader(ds.db_test), vlad=True, pca=None, gpu=args.gpu,
                                 rerank=args.rerank, rr_topk=args.rr_topk, lambda_value=args.lambda_value,
                                 nms=args.nms)
    synchronize()
    if args.rank == 0:
        print("RECALLS " + ",".join("%.6f" % r for r in recalls))
        if args.expect_recalls:
            want = np.array([float(v) for v in args.expect_recalls.split(",")])
            assert np.allclose(recalls, want), (recalls, want)
    torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()

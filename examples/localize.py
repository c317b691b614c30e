#!/usr/bin/env python
"""Localize query photos against a saved, device-resident place index.

Builds the index of the dataset's test gallery (dataset.db_test) with the model of --resume (and the PCA of
--pca-path), saves it to --index-dir, or loads it from there when it exists; then localizes dataset.q_test, prints
Recall@1/5/10 and writes <index-dir>/localize.csv: per query the top-10 gallery names, UTM positions and distances.

    python examples/localize.py -d pitts --scale 30k --data-dir data --resume logs/model_best.pth.tar --vlad \
        --pca-path logs/pca_params_model_best.h5 --features 4096 --index-dir logs/index
    python -m torch.distributed.run --nproc-per-node 8 examples/localize.py --launcher pytorch ...
"""
from __future__ import print_function, absolute_import

import argparse
import csv
import os
import os.path as osp
import sys

import torch
from torch.utils.data import DataLoader

sys.path.insert(0, osp.dirname(osp.dirname(osp.abspath(__file__))))

from ibl import datasets, models  # noqa: E402
from ibl.evaluators import recalls_from_topk  # noqa: E402
from ibl.index import PlaceIndex  # noqa: E402
from ibl.pca import PCA  # noqa: E402
from ibl.utils.data import get_transformer_test  # noqa: E402
from ibl.utils.data.preprocessor import Preprocessor  # noqa: E402
from ibl.utils.data.sampler import DistributedSliceSampler  # noqa: E402
from ibl.utils.dist_utils import init_dist, synchronize  # noqa: E402
from ibl.utils.serialization import copy_state_dict, load_checkpoint  # noqa: E402


def main():
    ap = argparse.ArgumentParser(description="Localize images against a place index")
    ap.add_argument("--launcher", type=str, choices=["none", "pytorch", "slurm"], default="none")
    ap.add_argument("--tcp-port", type=str, default="5017")
    ap.add_argument("-d", "--dataset", type=str, default="pitts", choices=datasets.names())
    ap.add_argument("--scale", type=str, default="30k")
    ap.add_argument("--data-dir", type=str, required=True)
    ap.add_argument("--resume", type=str, required=True)
    ap.add_argument("--vlad", action="store_true")
    ap.add_argument("--features", type=int, default=4096)
    ap.add_argument("--nowhiten", action="store_true")
    ap.add_argument("--pca-path", type=str, default=None, help="PCA parameters (ibl.pca.PCA); none: no PCA")
    ap.add_argument("--index-dir", type=str, required=True)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--test-batch-size", type=int, default=32)
    ap.add_argument("-j", "--workers", type=int, default=4)
    ap.add_argument("-k", type=int, default=10)
    args = ap.parse_args()
    args.gpu, args.rank = 0, 0
    if args.launcher != "none":
        init_dist(args.launcher, args)
        synchronize()
    torch.cuda.set_device(args.gpu)
    world = torch.distributed.get_world_size() if torch.distributed.is_initialized() else 1

    dataset = datasets.create(args.dataset, osp.join(args.data_dir, args.dataset), scale=args.scale)
    base = models.create("vgg16", pretrained=False)
    model = models.create("embednet", base, models.create("netvlad", dim=base.feature_dim)) if args.vlad else base
    copy_state_dict(load_checkpoint(args.resume)["state_dict"], model)
    model.cuda(args.gpu).eval()
    pca = None
    if args.pca_path:
        pca = PCA(args.features, not args.nowhiten, args.pca_path)

    if osp.isfile(osp.join(args.index_dir, "index.json")):
        index = PlaceIndex.load(args.index_dir, gpu=args.gpu, model=model)
        if args.rank == 0:
            print("loaded the place index of {} images from {}".format(index.n, args.index_dir))
    else:
        db_loader = DataLoader(
            Preprocessor(dataset.db_test, root=dataset.images_dir,
                         transform=get_transformer_test(args.height, args.width)),
            batch_size=args.test_batch_size, num_workers=args.workers,
            sampler=DistributedSliceSampler(dataset.db_test, num_replicas=world, rank=args.rank), shuffle=False,
            pin_memory=True)
        index = PlaceIndex.build(model, db_loader, dataset.db_test, pca=pca, vlad=args.vlad, gpu=args.gpu)
        index.save(args.index_dir)
        if args.rank == 0:
            print("built and saved the place index of {} images to {}".format(index.n, args.index_dir))

    # every rank localizes the same queries (the search is collective)
    q_loader = DataLoader(
        Preprocessor(dataset.q_test, root=dataset.images_dir,
                     transform=get_transformer_test(args.height, args.width, tokyo=(args.dataset == "tokyo"))),
        batch_size=(1 if args.dataset == "tokyo" else args.test_batch_size), num_workers=args.workers,
        shuffle=False, pin_memory=True)
    names = {it[0]: i for i, it in enumerate(index.gallery)}
    rows, ranked = [], []
    for imgs, fnames, _, _, _ in q_loader:
        for fname, places in zip(fnames, index.localize(imgs, k=args.k)):
            ranked.append([names[p[0]] for p in places] + [-1] * (args.k - len(places)))
            rows.append([fname] + [v for p in places for v in (p[0], p[2][0], p[2][1], repr(p[3]))])
    recalls = recalls_from_topk(ranked, dataset.test_pos, index.gallery, (1, 5, 10))
    if args.rank == 0:
        print("Recall Scores:")
        for i, kk in enumerate((1, 5, 10)):
            print("  top-{:<4}{:12.1%}".format(kk, recalls[i]))
        with open(osp.join(args.index_dir, "localize.csv"), "w", newline="") as f:
            w = csv.writer(f)
            w.writerow(["query"] + [c % (j + 1) for j in range(args.k) for c in ("name_%d", "x_%d", "y_%d", "dist_%d")])
            w.writerows(rows)


if __name__ == "__main__":
    main()

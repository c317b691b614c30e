#!/usr/bin/env python
"""Fine-tune the hub model (`hubconf.vgg16_netvlad()`: VGG16 -> NetVLAD(64) -> PCA-whitening 32768 -> 4096 -> L2) for a
few triplet steps on synthetic tuples under DistributedDataParallel, one process per rank.  There is no network, so the
model is built with pretrained=False and loaded with a synthetic state dict of the released model's shapes; everything
below conv5 is frozen as train_layers='conv5' freezes it (vgg.py:50-53).  Rank r trains on its own tuples (seed + r).

    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 examples/finetune_hub_synthetic.py

Ranks beyond the visible GPU count share GPUs over the gloo backend (NCCL takes one rank per GPU).  Prints one JSON
line from rank 0: the loss of every step, the device time of the last one, and whether every rank held identical
parameters after each optimizer step (the DDP invariant)."""
from __future__ import print_function, absolute_import

import argparse
import json
import os
import os.path as osp
import sys

import torch
import torch.nn.functional as F
from torch import nn

sys.path.insert(0, osp.dirname(osp.dirname(osp.abspath(__file__))))

from ibl import models  # noqa: E402
from openibl_b200 import synth  # noqa: E402


def build(args, gpu):
    base = models.create("vgg16", pretrained=False)
    model = models.create("embednetpca", base, models.create("netvlad", dim=base.feature_dim), dim=4096)
    model.load_state_dict(synth.make_state_dict(seed=args.seed, sharp=True, with_pca=True, bias_scale=0.02))
    for layer in list(model.base_model.base.children())[:24]:
        for p in layer.parameters():
            p.requires_grad = False
    model.cuda(gpu)
    return nn.parallel.DistributedDataParallel(model, device_ids=[gpu], output_device=gpu, find_unused_parameters=True)


def triplet(out, b, n, margin):
    """The reference Trainer._get_loss with loss_type='triplet' (ibl/trainers.py:81-94)."""
    out = out.view(b, n, -1)
    L = out.size(-1)
    neg = out[:, 2:]
    anc = out[:, 0].unsqueeze(1).expand_as(neg).contiguous().view(-1, L)
    pos = out[:, 1].unsqueeze(1).expand_as(neg).contiguous().view(-1, L)
    return F.triplet_margin_loss(anc, pos, neg.contiguous().view(-1, L), margin=margin, p=2, reduction="mean")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tuple-size", type=int, default=1)
    ap.add_argument("--neg-num", type=int, default=10)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--lr", type=float, default=0.001)
    ap.add_argument("--margin", type=float, default=0.1 ** 0.5)
    ap.add_argument("--seed", type=int, default=41)
    args = ap.parse_args()
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    gpu = int(os.environ.get("LOCAL_RANK", 0)) % torch.cuda.device_count()
    torch.cuda.set_device(gpu)
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29517")
    backend = "nccl" if world <= torch.cuda.device_count() else "gloo"
    torch.distributed.init_process_group(backend=backend, rank=rank, world_size=world)
    model = build(args, gpu)
    params = [p for p in model.parameters() if p.requires_grad]
    opt = torch.optim.SGD(params, lr=args.lr, momentum=0.9, weight_decay=0.001)
    n = 2 + args.neg_num
    easy, _ = synth.make_sfrs_tuples(seed=args.seed + rank, tuples=args.tuple_size, neg_num=args.neg_num, n_diff=1,
                                     height=args.height, width=args.width)
    x = easy.view(-1, 3, args.height, args.width).cuda(gpu)
    model.train()
    losses, identical, step_ms = [], [], 0.0
    for _ in range(args.steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        loss = triplet(model(x), args.tuple_size, n, args.margin)
        opt.zero_grad()
        loss.backward()
        opt.step()
        e1.record()
        torch.cuda.synchronize()
        step_ms = e0.elapsed_time(e1)
        losses.append(float(loss))
        chk = torch.stack([p.detach().double().sum() for p in params]).sum().reshape(1)
        allc = [torch.zeros_like(chk) for _ in range(world)]
        torch.distributed.all_gather(allc, chk)
        identical.append(bool(all(torch.equal(c, allc[0]) for c in allc)))
    if rank == 0:
        print("FINETUNE_HUB " + json.dumps({
            "world": world, "backend": backend, "tuple_size": args.tuple_size, "neg_num": args.neg_num,
            "image": [args.height, args.width], "losses_rank0": losses, "last_step_ms_rank0": step_ms,
            "params_identical_across_ranks_each_step": identical,
            "trainable_params": int(sum(p.numel() for p in params))}), flush=True)
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()

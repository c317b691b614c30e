#!/usr/bin/env python
"""Time one NetVLAD / SARE training step (`ibl.trainers.Trainer`, examples/netvlad_img.py): forward, backward and SGD
on a DistributedDataParallel-wrapped `EmbedNet` with the trunk frozen below conv5 (train_layers='conv5').

    python tools/bench_train.py                                   # 480x640, neg_num 10, tuple_size 1 and 4
    python tools/bench_train.py --tuple-sizes 4 --losses sare_ind --profile 10
    python -m torch.distributed.run --nproc-per-node 8 tools/bench_train.py

Each step feeds one tuple batch of (anchor, positive, neg_num negatives) per rank from pinned host memory, as the
recipe's DataLoader (pin_memory=True) does, so the host-to-device copy is part of the step.  Prints one JSON line:
per (tuple_size, loss) the ms/step and images/s of this rank (host clock around --steps steps that end in a device
synchronise, after --warmup steps), and the card name and power limit.  --profile N prints the N kernels with the
most device time over the timed steps of the last configuration (a separate run: the profiler slows the host)."""
import argparse
import json
import os
import socket
import subprocess
import sys
import time

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ibl import models  # noqa: E402
from ibl.trainers import Trainer  # noqa: E402
from openibl_b200 import synth  # noqa: E402


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                             "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = pl.stdout.strip() or None
    except Exception:
        power = None
    return name, power


def init_dist():
    """torch.distributed.run's environment when launched by it, else a one-process group on a free local port."""
    if "RANK" in os.environ:
        rank = int(os.environ["LOCAL_RANK"])
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl")
        return rank
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)
    return 0


class TupleLoader:
    """IterLoader's interface (new_epoch / next) over one fixed, pinned batch in the DataLoader's collated layout:
    a list over tuple positions of (images [tuple_size,3,H,W], fnames, pids, x, y)."""

    def __init__(self, tuple_size, neg_num, height, width, seed):
        n = 2 + neg_num
        imgs = synth.make_smooth_images(seed, tuple_size * n, height, width).view(tuple_size, n, 3, height, width)
        z = torch.zeros(tuple_size)
        self.batch = [(imgs[:, j].contiguous().pin_memory(), ["synthetic"] * tuple_size, z, z, z) for j in range(n)]

    def new_epoch(self):
        pass

    def next(self):
        return self.batch


def build_model(rank):
    base = models.create("vgg16", pretrained=False)
    m = models.create("embednet", base, models.create("netvlad", dim=512))
    m.load_state_dict(synth.make_state_dict(seed=7, sharp=True, with_pca=False, bias_scale=0.02))
    for layer in list(base.base.children())[:24]:          # what pretrained=True + train_layers='conv5' freezes
        for p in layer.parameters():
            p.requires_grad = False
    m.cuda(rank)
    return torch.nn.parallel.DistributedDataParallel(m, device_ids=[rank], output_device=rank,
                                                     find_unused_parameters=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--tuple-sizes", type=int, nargs="+", default=[1, 4])
    ap.add_argument("--losses", nargs="+", default=["triplet", "sare_ind"])
    ap.add_argument("--neg-num", type=int, default=10)
    ap.add_argument("--height", type=int, default=480)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile", type=int, default=0, metavar="N")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train.py needs a CUDA device (an H100): there is nothing to time without one")
    rank = init_dist()
    model = build_model(rank)
    opt = torch.optim.SGD(filter(lambda p: p.requires_grad, model.parameters()), lr=1e-4, momentum=0.9,
                          weight_decay=0.001)
    trainer = Trainer(model, margin=0.1 ** 0.5, gpu=rank)
    results, prof = [], None
    for tuple_size in args.tuple_sizes:
        loader = TupleLoader(tuple_size, args.neg_num, args.height, args.width, seed=100 + rank)
        for loss_type in args.losses:
            train = lambda steps: trainer.train(0, 0, loader, opt, train_iters=steps, print_freq=10 ** 9,
                                                vlad=True, loss_type=loss_type)
            train(args.warmup)
            torch.cuda.synchronize()
            dist.barrier()
            t0 = time.perf_counter()
            train(args.steps)
            torch.cuda.synchronize()
            ms = (time.perf_counter() - t0) * 1e3 / args.steps
            images = tuple_size * (2 + args.neg_num)
            results.append({"tuple_size": tuple_size, "loss": loss_type, "images_per_step": images,
                            "ms_per_step": round(ms, 3), "images_per_s": round(images * 1e3 / ms, 1)})
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            train(args.steps)
            torch.cuda.synchronize()
    name, power = card()
    if rank == 0:
        print(json.dumps({"bench": "trainer_step", "world_size": dist.get_world_size(),
                          "height": args.height, "width": args.width, "neg_num": args.neg_num, "steps": args.steps,
                          "warmup": args.warmup, "results": results, "gpu": name, "power_limit": power}))
        if prof is not None:
            print(prof.key_averages().table(sort_by="self_device_time_total", row_limit=args.profile), file=sys.stderr)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

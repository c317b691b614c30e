"""Seeded synthetic parameters, images and galleries for the hot path.

There is no network on the build or GPU boxes, so every benchmark / parity
input is generated from a seed.  The same generators feed the CUDA engine,
the CPU oracle and the golden-vector script, so all three see identical
bytes.  Shapes follow the reference:

  * VGG16 trunk conv1_1..conv5_3: 13 convs 3x3, state-dict slots
    {0,2,5,7,10,12,14,17,19,21,24,26,28} (reference ibl/models/vgg.py:40-42),
    kaiming-normal fan_out weights, zero bias (vgg.py:72-77).
  * NetVLAD K=64 (any 1..64 on request), C=512: centroids ~ U[0,1) (netvlad.py:29); conv weight
    default Conv2d init; the "sharp" variant mimics _init_params
    (netvlad.py:34-42) with alpha from the top-2 dot gap.
  * PCA layer Conv2d(K*512, 4096, 1) default init (netvlad.py:89).
"""
from __future__ import annotations

import math
from collections import OrderedDict

import numpy as np
import torch

# (state-dict slot, Cin, Cout) for the 13 convs; 'P' marks a 2x2 max-pool.
VGG16_PLAN = [
    (0, 3, 64), (2, 64, 64), "P",
    (5, 64, 128), (7, 128, 128), "P",
    (10, 128, 256), (12, 256, 256), (14, 256, 256), "P",
    (17, 256, 512), (19, 512, 512), (21, 512, 512), "P",
    (24, 512, 512), (26, 512, 512), (28, 512, 512),
]
VGG16_CONV_SLOTS = [p[0] for p in VGG16_PLAN if p != "P"]


def _gen(seed: int) -> torch.Generator:
    g = torch.Generator(device="cpu")
    g.manual_seed(int(seed))
    return g


def make_vgg_weights(seed: int = 0, bias_scale: float = 0.0) -> "OrderedDict[str, torch.Tensor]":
    """13 (weight, bias) pairs keyed like the reference state dict ('base.N.weight').

    bias_scale=0 reproduces reset_params (zero bias); tests also use a non-zero
    bias so the bias path of the kernels is exercised."""
    g = _gen(seed)
    sd = OrderedDict()
    for item in VGG16_PLAN:
        if item == "P":
            continue
        slot, cin, cout = item
        std = math.sqrt(2.0 / (cout * 9))  # kaiming_normal_, mode='fan_out'
        sd[f"base.{slot}.weight"] = torch.randn(cout, cin, 3, 3, generator=g) * std
        if bias_scale:
            sd[f"base.{slot}.bias"] = torch.randn(cout, generator=g) * bias_scale
        else:
            sd[f"base.{slot}.bias"] = torch.zeros(cout)
    return sd


def make_netvlad_params(seed: int = 0, num_clusters: int = 64, dim: int = 512, sharp: bool = False):
    """Returns dict(centroids [K,C], conv_weight [K,C,1,1], alpha)."""
    g = _gen(seed + 1000)
    if not sharp:
        bound = 1.0 / math.sqrt(dim)  # Conv2d default (kaiming_uniform a=sqrt(5))
        conv_w = (torch.rand(num_clusters, dim, 1, 1, generator=g) * 2 - 1) * bound
        cent = torch.rand(num_clusters, dim, generator=g)
        return {"centroids": cent, "conv_weight": conv_w, "alpha": 100.0}
    # _init_params-style: unit-norm cluster centres and train descriptors
    clsts = torch.randn(num_clusters, dim, generator=g)
    clsts = clsts / clsts.norm(dim=1, keepdim=True)
    desc = torch.randn(5000, dim, generator=g)
    desc = desc / desc.norm(dim=1, keepdim=True)
    clsts_n = clsts.numpy().astype(np.float32)
    assign = clsts_n / np.linalg.norm(clsts_n, axis=1, keepdims=True)
    dots = assign @ desc.numpy().T
    dots.sort(0)
    dots = dots[::-1, :]
    # one cluster has no runner-up to set alpha by; its assignment is 1 whatever alpha is
    alpha = float(-np.log(0.01) / np.mean(dots[0, :] - dots[1, :])) if num_clusters > 1 else 100.0
    conv_w = torch.from_numpy((alpha * assign).astype(np.float32)).reshape(num_clusters, dim, 1, 1)
    return {"centroids": torch.from_numpy(clsts_n.copy()), "conv_weight": conv_w, "alpha": alpha}


def make_pca_params(seed: int = 0, in_dim: int = 32768, out_dim: int = 4096):
    """Conv2d(in_dim, out_dim, 1) default init: weight, bias ~ U(-1/sqrt(in), 1/sqrt(in))."""
    g = _gen(seed + 2000)
    bound = 1.0 / math.sqrt(in_dim)
    w = torch.empty(out_dim, in_dim, 1, 1)
    w.uniform_(-bound, bound, generator=g)
    b = torch.empty(out_dim)
    b.uniform_(-bound, bound, generator=g)
    return {"weight": w, "bias": b}


def make_state_dict(seed: int = 0, sharp: bool = False, with_pca: bool = True,
                    pca_dim: int = 4096, bias_scale: float = 0.0, num_clusters: int = 64):
    """Full EmbedNet / EmbedNetPCA state dict with the reference's key names
    (SURVEY 8b: base_model.base.N.*, net_vlad.*, pca_layer.*) for a NetVLAD layer of
    `num_clusters` clusters; the PCA layer's input is num_clusters * 512."""
    sd = OrderedDict()
    for k, v in make_vgg_weights(seed, bias_scale).items():
        sd["base_model." + k] = v
    nv = make_netvlad_params(seed, num_clusters=num_clusters, sharp=sharp)
    sd["net_vlad.centroids"] = nv["centroids"]
    sd["net_vlad.conv.weight"] = nv["conv_weight"]
    if with_pca:
        p = make_pca_params(seed, num_clusters * 512, pca_dim)
        sd["pca_layer.weight"] = p["weight"]
        sd["pca_layer.bias"] = p["bias"]
    return sd


def make_images(seed: int, batch: int, height: int = 480, width: int = 640) -> torch.Tensor:
    """randn images, NCHW fp32 (SURVEY 8d)."""
    return torch.randn(batch, 3, height, width, generator=_gen(seed))


def make_smooth_images(seed: int, batch: int, height: int, width: int, amp: float = 2.0) -> torch.Tensor:
    """Smooth random fields (a 3 x H/16 x W/16 normal sample upsampled bilinearly): unlike white noise they give
    clearly different descriptors through a random-init trunk (used where similarities must not all be ~1)."""
    c = torch.randn(batch, 3, max(height // 16, 2), max(width // 16, 2), generator=_gen(seed))
    return torch.nn.functional.interpolate(c, size=(height, width), mode="bilinear", align_corners=False) * amp


def make_sfrs_tuples(seed: int, tuples: int, neg_num: int, n_diff: int, height: int, width: int):
    """(inputs_easy [B, neg_num+2, 3,H,W], inputs_diff [B, 1+n_diff, 3,H,W]) as SFRSTrainer._parse_data produces them
    (trainers.py:228-233): anchor, its positive (anchor + noise), negatives (other places); the difficult positives
    are noisier views of the anchor."""
    g = _gen(seed + 77)
    per = 1 + neg_num
    fields = make_smooth_images(seed, tuples * per, height, width).view(tuples, per, 3, height, width)
    noise = lambda s: s * torch.randn(tuples, 3, height, width, generator=g)
    anchor = fields[:, 0]
    negs = []
    for i in range(neg_num):           # negative i: another place whose quadrant i % 4 shows the anchor's scene, so its
        n = fields[:, 1 + i].clone()   # best-matching REGION is a quarter, not the whole image (exercises trainers.py:261-271)
        h0, w0 = (i % 4 // 2) * (height // 2), (i % 2) * (width // 2)
        n[:, :, h0:h0 + height // 2, w0:w0 + width // 2] = anchor[:, :, h0:h0 + height // 2, w0:w0 + width // 2]
        negs.append(n)
    easy = torch.stack([anchor, anchor + noise(0.4)] + negs, dim=1)
    diff = torch.stack([anchor] + [anchor + noise(0.9) for _ in range(n_diff)], dim=1)
    return easy.contiguous(), diff.contiguous()


def make_gallery(n_db: int, n_q: int, dim: int = 4096, sigma: float = 0.25,
                 seed_db: int = 2, seed_q: int = 3):
    """Pitts-shaped synthetic retrieval set (SURVEY 8d).

    db rows are unit-norm randn; query q is normalize(db[gt[q]] + sigma*randn), so the
    planted positive is usually, but not always, the nearest neighbour.
    Returns (q [n_q,dim], db [n_db,dim], gt int64 [n_q])."""
    gd, gq = _gen(seed_db), _gen(seed_q)
    db = torch.randn(n_db, dim, generator=gd)
    db = db / db.norm(dim=1, keepdim=True)
    gt = torch.randint(0, n_db, (n_q,), generator=gq)
    q = db[gt] + sigma * torch.randn(n_q, dim, generator=gq)
    q = q / q.norm(dim=1, keepdim=True)
    return q.contiguous(), db.contiguous(), gt

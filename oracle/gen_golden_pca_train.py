#!/usr/bin/env python
"""Golden vectors for one EmbedNetPCA fine-tuning step: the UNMODIFIED reference `EmbedNetPCA`
(ibl/models/netvlad.py:84-110) in train mode on CPU, a triplet loss on its output as the reference `Trainer._get_loss`
computes it (ibl/trainers.py:81-94, margin 0.1 ** 0.5 as netvlad_img.py:169 passes it), and `loss.backward()`, with
everything below conv5 frozen as `pretrained=True, train_layers='conv5'` freezes it (vgg.py:50-53).  Synthetic weights
with 8 clusters and a 64-d PCA layer (D = 4096) keep the fixture near 1 MB.  Recorded: the loss, the output, the full
gradients of pca_layer.weight / bias, net_vlad.conv.weight and centroids, the conv5 bias gradients, and 16 seeded
random projections of each conv5 weight gradient (the full ones are ~28 MB).  TEST INFRASTRUCTURE; build container
only (needs /root/reference).

    python oracle/gen_golden_pca_train.py     # writes tests/golden/pca_train.npz
"""
import os, sys, types, warnings
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.modules.setdefault("h5py", types.ModuleType("h5py"))
sys.path.insert(0, os.environ.get("IBL_REFERENCE", "/root/reference"))
warnings.filterwarnings("ignore")
from ibl import models as ref_models          # the reference's ibl
from ibl.trainers import Trainer              # the reference's trainer
from oracle.gen_golden_trainer import write_npz
from openibl_b200 import synth

B, NEG, H, W, SEED, K, PCA_DIM = 2, 2, 64, 96, 21, 8, 64
MARGIN = 0.1 ** 0.5
CONV5 = (24, 26, 28)
N_PROJ = 16


def make_inputs():
    """[B, 2 + NEG, 3, H, W]: anchor, positive (anchor + noise), NEG negatives."""
    easy, _ = synth.make_sfrs_tuples(seed=43, tuples=B, neg_num=NEG, n_diff=1, height=H, width=W)
    return easy


def make_state_dict():
    return synth.make_state_dict(seed=SEED, sharp=True, with_pca=True, num_clusters=K, pca_dim=PCA_DIM, bias_scale=0.02)


def projections(slot, numel):
    """[N_PROJ, numel] fp64 random directions for the weight gradient of conv `slot` (the test recomputes them)."""
    g = torch.Generator().manual_seed(1000 + slot)
    return torch.randn(N_PROJ, numel, generator=g, dtype=torch.float64)


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(4)                 # fixed: the CPU convolutions' summation order follows the thread count
    x = make_inputs()
    base = ref_models.create("vgg16", pretrained=False)
    model = ref_models.create("embednetpca", base, ref_models.create("netvlad", num_clusters=K, dim=512), dim=PCA_DIM)
    model.load_state_dict(make_state_dict())
    for layer in list(model.base_model.base.children())[:24]:
        for p in layer.parameters():
            p.requires_grad = False
    model.train()
    out = model(x.view(-1, 3, H, W))
    loss = Trainer(None, margin=MARGIN, gpu=None)._get_loss(out, "triplet", B, 2 + NEG)
    loss.backward()
    res = dict(loss=np.float64(loss.item()), out=out.detach().numpy(),
               grad_pca_w=model.pca_layer.weight.grad.numpy(), grad_pca_b=model.pca_layer.bias.grad.numpy(),
               grad_conv_w=model.net_vlad.conv.weight.grad.numpy(), grad_centroids=model.net_vlad.centroids.grad.numpy())
    for slot in CONV5:
        conv = model.base_model.base[slot]
        gw = conv.weight.grad.double().reshape(-1)
        res[f"proj_w{slot}"] = (projections(slot, gw.numel()) @ gw).numpy()
        res[f"grad_b{slot}"] = conv.bias.grad.numpy()
    assert model.base_model.base[21].weight.grad is None
    path = os.path.join(ROOT, "tests", "golden", "pca_train.npz")
    write_npz(path, res)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB", "loss", loss.item(), "out", tuple(out.shape))

#!/usr/bin/env python
"""Golden vectors for NetVLAD layers of fewer than 64 clusters, `NetVLAD(num_clusters=K, dim=512)` as the reference
constructs it (ibl/models/netvlad.py:11-29), all from the UNMODIFIED reference modules on CPU:

* raw NetVLAD [B,K,512] and EmbedNet descriptors [B,K*512] for K in {1, 8, 32, 48, 63}, `_init_params`-style
  (sharp) parameters, at 64x96 (24 feature pixels) and at 240x320 (300 feature pixels, three 128-pixel tiles);
* EmbedNetPCA descriptors at K = 32 with a seeded PCA layer of input 32*512;
* one `Trainer._forward` triplet step at K = 32 (ibl/trainers.py:70-162), recorded as gen_golden_trainer.py does;
* one `SFRSTrainer._forward` region step at K = 16, generation 1 (ibl/trainers.py:235-259), recorded as
  gen_golden_sfrs.py does.

TEST INFRASTRUCTURE; build container only (needs /root/reference).

    python oracle/gen_golden_clusters.py     # writes tests/golden/clusters.npz
"""
import os, sys, types, warnings
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.modules.setdefault("h5py", types.ModuleType("h5py"))
sys.path.insert(0, os.environ.get("IBL_REFERENCE", "/root/reference"))
warnings.filterwarnings("ignore")
from ibl import models as ref_models          # the reference's ibl
from ibl.trainers import SFRSTrainer, Trainer  # the reference's trainers
from openibl_b200 import synth
from gen_golden_trainer import write_npz

KS = (1, 8, 32, 48, 63)
# (tag, batch, H, W, image seed)
SIZES = (("s", 2, 64, 96, 21), ("l", 1, 240, 320, 22))
SEED = 17                                    # model parameters; the NetVLAD draws depend on K
PCA_K, PCA_DIM = 32, 128
TRAIN_K, SFRS_K = 32, 16


def model_sd(K, seed=SEED, with_pca=False, bias_scale=0.05):
    return synth.make_state_dict(seed=seed, sharp=True, with_pca=with_pca, pca_dim=PCA_DIM, bias_scale=bias_scale,
                                 num_clusters=K)


def netvlad(K):
    return ref_models.create("netvlad", num_clusters=K, dim=512)


def freeze_below_conv5(trunk):
    for layer in list(trunk.base.children())[:24]:       # what pretrained=True + train_layers='conv5' freezes
        for p in layer.parameters():
            p.requires_grad = False


@torch.no_grad()
def descriptors(out):
    for tag, b, h, w, img_seed in SIZES:
        x = synth.make_images(seed=img_seed, batch=b, height=h, width=w)
        for K in KS:
            m = ref_models.create("embednet", ref_models.create("vgg16", pretrained=False), netvlad(K))
            m.load_state_dict(model_sd(K), strict=True)
            m.eval()
            _, feat = m.base_model(x)
            raw = m.net_vlad(feat)
            _, vlad = m(x)
            assert raw.shape == (b, K, 512) and vlad.shape == (b, K * 512)
            out[f"{tag}_k{K}_raw"] = raw[:, :, ::8].numpy().copy()
            out[f"{tag}_k{K}_vlad"] = vlad[:, ::4].numpy().copy()
            print(f"{tag} K={K}: |raw| {raw.norm():.4f}")
    tag, b, h, w, img_seed = SIZES[0]
    x = synth.make_images(seed=img_seed, batch=b, height=h, width=w)
    m = ref_models.create("embednetpca", ref_models.create("vgg16", pretrained=False), netvlad(PCA_K), dim=PCA_DIM)
    m.load_state_dict(model_sd(PCA_K, with_pca=True), strict=True)
    out[f"pca_k{PCA_K}_desc"] = m.eval()(x).numpy().copy()


def trainer_step(out):
    """gen_golden_trainer.py's triplet case on the VLAD descriptor, with TRAIN_K clusters."""
    easy, _ = synth.make_sfrs_tuples(seed=41, tuples=2, neg_num=3, n_diff=1, height=64, width=96)
    m = ref_models.create("embednet", ref_models.create("vgg16", pretrained=False), netvlad(TRAIN_K))
    m.load_state_dict(model_sd(TRAIN_K, seed=13, bias_scale=0.02))
    freeze_below_conv5(m.base_model)
    m.train()
    loss = Trainer(m, margin=0.1 ** 0.5, gpu=None)._forward(easy.clone(), True, "triplet")
    loss.backward()
    out["train_loss"] = np.float64(loss.item())
    for slot in (24, 26, 28):
        conv = m.base_model.base[slot]
        out[f"train_w{slot}"] = conv.weight.grad.numpy()[::16, ::8].copy()
        out[f"train_b{slot}"] = conv.bias.grad.numpy().copy()
        out[f"train_w{slot}_norm"] = np.float64(conv.weight.grad.double().norm().item())
    out["train_centroids"] = m.net_vlad.centroids.grad.numpy()[:, ::4].copy()
    out["train_conv_w"] = m.net_vlad.conv.weight.grad.numpy()[:, ::4, 0, 0].copy()
    print(f"trainer K={TRAIN_K}: loss {loss.item():.6f}")


def sfrs_step(out):
    """gen_golden_sfrs.py's generation-1 step (hard-region loss + soft loss), with SFRS_K clusters; the reference runs
    one tuple at a time (tuple_size 1) and the B tuples are averaged."""
    B, NEG, NDIFF = 2, 2, 2

    def build(seed):
        m = ref_models.create("embedregionnet", ref_models.create("vgg16", pretrained=False), netvlad(SFRS_K),
                              tuple_size=1)
        m.load_state_dict(model_sd(SFRS_K, seed=seed, bias_scale=0.02))
        freeze_below_conv5(m.base_model)
        return m.train()

    easy, diff = synth.make_sfrs_tuples(seed=31, tuples=B, neg_num=NEG, n_diff=NDIFF, height=64, width=96)
    model, cache = build(13), build(23)
    tr = SFRSTrainer(model, cache, margin=0.1, neg_num=NEG, gpu=None, temp=[0.07, 0.07])
    hard, soft = 0.0, 0.0
    for t in range(B):
        lh, ls = tr._forward(easy[t:t + 1], diff[t:t + 1], "sare_ind", 1)
        ((lh + 0.5 * ls) / B).backward()
        hard += lh.item() / B
        soft += ls.item() / B
    out["sfrs_loss_hard"], out["sfrs_loss_soft"] = np.float64(hard), np.float64(soft)
    for slot in (24, 26, 28):
        conv = model.base_model.base[slot]
        out[f"sfrs_w{slot}"] = conv.weight.grad.numpy()[::8, ::8].copy()
        out[f"sfrs_b{slot}"] = conv.bias.grad.numpy().copy()
        out[f"sfrs_w{slot}_norm"] = np.float64(conv.weight.grad.double().norm().item())
    out["sfrs_centroids"] = model.net_vlad.centroids.grad.numpy()[:, ::4].copy()
    out["sfrs_conv_w"] = model.net_vlad.conv.weight.grad.numpy()[:, ::4, 0, 0].copy()
    print(f"sfrs K={SFRS_K}: loss_hard {hard:.6f} loss_soft {soft:.6f}")


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(4)                 # fixed: the CPU convolutions' summation order follows the thread count
    out = {}
    descriptors(out)
    trainer_step(out)
    sfrs_step(out)
    path = os.path.join(ROOT, "tests", "golden", "clusters.npz")
    write_npz(path, out)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")

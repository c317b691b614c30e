"""One EmbedNetPCA fine-tuning step restated with oracle/ibl_oracle.py, pinned against the unmodified reference
(tests/golden/pca_train.npz, oracle/gen_golden_pca_train.py).  `pca_train_step` is also the fp64 yardstick of the GPU
tests in test_gpu_pca_train.py."""
import numpy as np
import torch
import torch.nn.functional as F

from conftest import load_golden, rel_l2
from oracle import ibl_oracle as O
from openibl_b200 import synth

B, NEG, H, W, SEED, K, PCA_DIM = 2, 2, 64, 96, 21, 8, 64      # as oracle/gen_golden_pca_train.py
MARGIN = 0.1 ** 0.5
CONV5 = (24, 26, 28)
N_PROJ = 16


def golden_inputs():
    easy, _ = synth.make_sfrs_tuples(seed=43, tuples=B, neg_num=NEG, n_diff=1, height=H, width=W)
    sd = synth.make_state_dict(seed=SEED, sharp=True, with_pca=True, num_clusters=K, pca_dim=PCA_DIM, bias_scale=0.02)
    return easy, sd


def projections(slot, numel):
    g = torch.Generator().manual_seed(1000 + slot)
    return torch.randn(N_PROJ, numel, generator=g, dtype=torch.float64)


def triplet_loss(out, b, n, margin=MARGIN):
    """The reference Trainer._get_loss, loss_type='triplet' (ibl/trainers.py:81-94)."""
    out = out.view(b, n, -1)
    L = out.size(-1)
    neg = out[:, 2:]
    anc = out[:, 0].unsqueeze(1).expand_as(neg).contiguous().view(-1, L)
    pos = out[:, 1].unsqueeze(1).expand_as(neg).contiguous().view(-1, L)
    return F.triplet_margin_loss(anc, pos, neg.contiguous().view(-1, L), margin=margin, p=2, reduction="mean")


def pca_train_step(sd, x, b, n, trainable, dtype=torch.float64, device="cpu"):
    """EmbedNetPCA forward (netvlad.py:95-110) + triplet loss + backward on the oracle's functions.
    -> (loss, out, {name: grad}) for the state-dict keys in `trainable`."""
    p = {k: v.to(device=device, dtype=dtype).requires_grad_(k in trainable) for k, v in sd.items()}
    feat = O.vgg16_trunk(x.to(device=device, dtype=dtype), p)
    v = O.vlad_normalize(O.netvlad(feat, p["net_vlad.conv.weight"], p["net_vlad.centroids"]))
    out = O.pca_whiten(v, p["pca_layer.weight"], p["pca_layer.bias"])
    loss = triplet_loss(out, b, n)
    loss.backward()
    return loss.detach(), out.detach(), {k: p[k].grad for k in trainable}


def conv5_and_head():
    return [f"base_model.base.{s}.{t}" for s in CONV5 for t in ("weight", "bias")] + \
           ["net_vlad.conv.weight", "net_vlad.centroids", "pca_layer.weight", "pca_layer.bias"]


def check_against_golden(loss, out, grads, tol):
    """grads: state-dict key -> gradient (any float tensor); every check is a relative L2 error below `tol`."""
    g = load_golden("pca_train")
    errs = {"loss": abs(float(loss) - float(g["loss"])) / abs(float(g["loss"])), "out": rel_l2(out, g["out"]),
            "pca_w": rel_l2(grads["pca_layer.weight"], g["grad_pca_w"]),
            "pca_b": rel_l2(grads["pca_layer.bias"], g["grad_pca_b"]),
            "conv_w": rel_l2(grads["net_vlad.conv.weight"], g["grad_conv_w"]),
            "centroids": rel_l2(grads["net_vlad.centroids"], g["grad_centroids"])}
    for s in CONV5:
        gw = grads[f"base_model.base.{s}.weight"].double().reshape(-1).cpu()
        errs[f"w{s}"] = rel_l2(projections(s, gw.numel()) @ gw, g[f"proj_w{s}"])
        errs[f"b{s}"] = rel_l2(grads[f"base_model.base.{s}.bias"], g[f"grad_b{s}"])
    bad = {k: v for k, v in errs.items() if not v < tol}
    assert not bad, (bad, errs)
    return errs


def test_oracle_pca_train_step_matches_reference():
    """Same torch CPU kernels in fp32 in a different op order (NetVLAD, the PCA matmul): rounding only."""
    x, sd = golden_inputs()
    loss, out, grads = pca_train_step(sd, x.view(-1, 3, H, W), B, 2 + NEG, conv5_and_head(), dtype=torch.float32)
    check_against_golden(loss, out, grads, 2e-5)


def test_golden_step_is_a_real_triplet_step():
    """The recorded step is informative: the loss is active and every recorded gradient is nonzero."""
    g = load_golden("pca_train")
    assert 0.0 < float(g["loss"]) < 2 * MARGIN
    for k in ("grad_pca_w", "grad_pca_b", "grad_conv_w", "grad_centroids", "proj_w28", "grad_b24"):
        assert np.abs(g[k]).max() > 0, k
    assert g["grad_pca_w"].shape == (PCA_DIM, K * 512, 1, 1)

#!/usr/bin/env python
"""Golden vectors for one NetVLAD / SARE training step (examples/netvlad_img.py): the UNMODIFIED reference
`Trainer._forward` (ibl/trainers.py:70-162) driving the UNMODIFIED reference `EmbedNet` (ibl/models/netvlad.py:63-82)
on CPU, with the trunk frozen below conv5 as `pretrained=True, train_layers='conv5'` freezes it (vgg.py:50-53), and
`margin = 0.1 ** 0.5` as netvlad_img.py:169 passes it.  Cases: loss_type in {triplet, sare_ind, sare_joint} on the
VLAD descriptor, and triplet with vlad=False -- the max-pool branch, where the model is the bare `VGG` and the loss
is on `pool_x`.  TEST INFRASTRUCTURE; build container only (needs /root/reference).

    python oracle/gen_golden_trainer.py     # writes tests/golden/trainer_step.npz
"""
import io, os, sys, types, warnings, zipfile
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.modules.setdefault("h5py", types.ModuleType("h5py"))
sys.path.insert(0, os.environ.get("IBL_REFERENCE", "/root/reference"))
warnings.filterwarnings("ignore")
from ibl import models as ref_models          # the reference's ibl
from ibl.trainers import Trainer              # the reference's trainer
from openibl_b200 import synth

B, NEG, H, W, SEED = 2, 3, 64, 96, 13
MARGIN = 0.1 ** 0.5
CASES = [("triplet", True), ("sare_ind", True), ("sare_joint", True), ("triplet", False)]
# (B, N, scale) of the loss-only cases: unit-norm rows (VLAD-like) when scale is None, else randn * scale (pool-like)
LOSS_SHAPES = [(1, 3, None), (2, 5, None), (4, 12, None), (3, 4, 0.2)]


def case_name(loss_type, vlad):
    return f"{loss_type}_{'vlad' if vlad else 'pool'}"


def make_inputs():
    """[B, 2 + NEG, 3, H, W]: anchor, positive (anchor + noise), NEG negatives (other places sharing one quadrant)."""
    easy, _ = synth.make_sfrs_tuples(seed=41, tuples=B, neg_num=NEG, n_diff=1, height=H, width=W)
    return easy


def build(vlad):
    base = ref_models.create("vgg16", pretrained=False)
    if vlad:
        m = ref_models.create("embednet", base, ref_models.create("netvlad", dim=512))
        m.load_state_dict(synth.make_state_dict(seed=SEED, sharp=True, with_pca=False, bias_scale=0.02))
        trunk = m.base_model
    else:
        m = base
        m.load_state_dict(synth.make_vgg_weights(SEED, 0.02))
        trunk = m
    for layer in list(trunk.base.children())[:24]:          # what pretrained=True + train_layers='conv5' freezes
        for p in layer.parameters():
            p.requires_grad = False
    return m.train(), trunk


def write_npz(path, arrays):
    """np.savez_compressed with fixed member timestamps, so that a rerun writes the same bytes."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
        for key in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[key]), allow_pickle=False)
            info = zipfile.ZipInfo(key + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(4)                 # fixed: the CPU convolutions' summation order follows the thread count
    x = make_inputs()
    out = {}
    for loss_type, vlad in CASES:
        name = case_name(loss_type, vlad)
        model, trunk = build(vlad)
        loss = Trainer(model, margin=MARGIN, gpu=None)._forward(x.clone(), vlad, loss_type)
        loss.backward()
        out[f"{name}_loss"] = np.float64(loss.item())
        for slot in (24, 26, 28):
            conv = trunk.base[slot]
            out[f"{name}_w{slot}"] = conv.weight.grad.numpy()[::16, ::8].copy()
            out[f"{name}_b{slot}"] = conv.bias.grad.numpy().copy()
            out[f"{name}_w{slot}_norm"] = np.float64(conv.weight.grad.double().norm().item())
        if vlad:
            out[f"{name}_centroids"] = model.net_vlad.centroids.grad.numpy()[:, ::4].copy()
            out[f"{name}_conv_w"] = model.net_vlad.conv.weight.grad.numpy()[:, ::4, 0, 0].copy()
        assert trunk.base[21].weight.grad is None
        print(f"{name}: loss {loss.item():.6f}  |dW28| {out[f'{name}_w28_norm']:.3e}")
    # the loss algebra alone: reference _get_loss and its gradient on random descriptors, several (B, N)
    g = torch.Generator().manual_seed(5)
    tr = Trainer(None, margin=MARGIN, gpu=None)
    for (b, n, scale) in LOSS_SHAPES:
        d = torch.randn(b * n, 64, generator=g)
        d = torch.nn.functional.normalize(d, dim=1) if scale is None else d * scale
        out[f"u{b}x{n}_outputs"] = d.numpy()
        for lt in ("triplet", "sare_ind", "sare_joint"):
            o = d.clone().requires_grad_(True)
            loss = tr._get_loss(o, lt, b, n)
            loss.backward()
            out[f"u{b}x{n}_{lt}_loss"] = np.float64(loss.item())
            out[f"u{b}x{n}_{lt}_grad"] = o.grad.numpy().copy()
    path = os.path.join(ROOT, "tests", "golden", "trainer_step.npz")
    write_npz(path, out)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")

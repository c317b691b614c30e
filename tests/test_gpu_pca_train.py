"""Fine-tuning EmbedNetPCA end to end: the PCA layer's training forward and backward (ibl_pca_forward_train /
ibl_pca_backward: tensor-core dgrad and wgrad kernels, CUDA-core fp32 in the other math mode) against fp64 torch, the
model's training step against the unmodified reference (tests/golden/pca_train.npz) and against an fp64 restatement
(test_host_pca_train.pca_train_step), frozen parts, a few SGD steps, and the eval path afterwards.  The SASS check at
the end needs no GPU."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import rel_l2
from openibl_b200 import synth
from test_host_pca_train import (B, H, K, NEG, PCA_DIM, W, check_against_golden, conv5_and_head, golden_inputs,
                                 pca_train_step, triplet_loss)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "openibl_b200", "lib", "libiblb200.so")
SENTINEL = 1234.5
GUARD = 4096


@pytest.fixture(scope="module")
def eng():
    from openibl_b200.engine import Engine
    e = Engine.get(0)
    yield e
    e.set_gemm_mode(1)
    e.conv_mode = 1


def _modes():
    from openibl_b200.engine import CONV_SIMT_FP32, CONV_TC_BF16X3
    return {"tc": CONV_TC_BF16X3, "simt": CONV_SIMT_FP32}


def _guarded(n):
    buf = torch.full((n + GUARD,), SENTINEL, device="cuda")
    return buf, buf[:n]


ABI_CASES = [(n, 4096, 32768) for n in (1, 12, 48, 97)] + [(n, 200, 512) for n in (1, 12, 48, 97)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["tc", "simt"])
@pytest.mark.parametrize("case", ABI_CASES, ids=lambda c: f"N{c[0]}_P{c[1]}_D{c[2]}")
def test_pca_train_abi_vs_fp64(eng, mode, case):
    """y = v W^T + b, gv = gy W, gW = gy^T v, gb = sum gy through the C ABI against fp64 torch, and the guard regions
    behind gv, gW and gb keep their sentinel."""
    from openibl_b200._cabi import check
    from openibl_b200.engine import _ptr, _stream
    N, P, D = case
    g = torch.Generator(device="cuda").manual_seed(N * 7 + P)
    v = torch.nn.functional.normalize(torch.randn(N, D, device="cuda", generator=g), dim=1)
    Wt = (torch.rand(P, D, device="cuda", generator=g) * 2 - 1) / D ** 0.5
    b = (torch.rand(P, device="cuda", generator=g) * 2 - 1) / D ** 0.5
    gy = torch.randn(N, P, device="cuda", generator=g)
    eng.set_gemm_mode(_modes()[mode])
    eng.set_pca(Wt, b, force=True)
    y = eng.pca_forward_train(v, Wt, b)
    gv_buf, gv = _guarded(N * D)
    gw_buf, gw = _guarded(P * D)
    gb_buf, gb = _guarded(P)
    check(eng.lib.ibl_pca_backward(eng.h, _ptr(v), N, D, _ptr(Wt), P, _ptr(gy), _ptr(gv), _ptr(gw), _ptr(gb),
                                   _stream(0)), "ibl_pca_backward")
    torch.cuda.synchronize()
    vd, Wd, gyd = v.double(), Wt.double(), gy.double()
    yd = vd @ Wd.t() + b.double()
    errs = {"y": float((y.double() - yd).norm() / yd.norm()),
            "gv": float((gv.view(N, D).double() - gyd @ Wd).norm() / (gyd @ Wd).norm()),
            "gW": float((gw.view(P, D).double() - gyd.t() @ vd).norm() / (gyd.t() @ vd).norm()),
            "gb": float((gb.double() - gyd.sum(0)).norm() / gyd.sum(0).norm())}
    print(mode, case, errs)
    # y comes from the inference GEMM (the forward shares it with extraction): random W makes |y| small against its
    # terms, and the bf16x3 split-K sums measure up to 2e-5 there; the backward GEMMs hold 1e-5
    assert errs["y"] <= 5e-5 and all(errs[k] <= 1e-5 for k in ("gv", "gW", "gb")), errs
    for name, buf, n in (("gv", gv_buf, N * D), ("gW", gw_buf, P * D), ("gb", gb_buf, P)):
        assert bool((buf[n:] == SENTINEL).all()), f"{name} guard overwritten"


@pytest.mark.gpu
def test_pca_backward_optional_outputs_and_errors(eng):
    """gv / gW / gb may each be NULL; the tensor-core path refuses a W whose planes the engine does not hold."""
    from openibl_b200._cabi import IblError
    N, P, D = 12, 256, 1024
    g = torch.Generator(device="cuda").manual_seed(3)
    v, Wt = torch.randn(N, D, device="cuda", generator=g), torch.randn(P, D, device="cuda", generator=g)
    b, gy = torch.randn(P, device="cuda", generator=g), torch.randn(N, P, device="cuda", generator=g)
    eng.set_gemm_mode(_modes()["tc"])
    eng.set_pca(Wt, b, force=True)
    gv_all, gw_all, gb_all = eng.pca_backward(v, Wt, gy)
    gv, gw, gb = eng.pca_backward(v, Wt, gy, need_gv=False, need_gb=False)
    assert gv is None and gb is None and torch.equal(gw, gw_all)
    gv, gw, gb = eng.pca_backward(None, Wt, gy, need_gw=False)
    assert gw is None and torch.equal(gv, gv_all) and torch.equal(gb, gb_all)
    other = Wt.clone()
    with pytest.raises(IblError, match="ibl_engine_set_pca"):
        eng.pca_backward(v, other, gy)
    with pytest.raises(IblError, match="ibl_engine_set_pca"):
        eng.pca_forward_train(v, other, b)


def _model(sd, num_clusters, pca_dim, freeze_below_conv5=True):
    from ibl import models
    base = models.create("vgg16", pretrained=False)
    m = models.create("embednetpca", base, models.create("netvlad", num_clusters=num_clusters, dim=512), dim=pca_dim)
    m.load_state_dict(sd)
    if freeze_below_conv5:
        for layer in list(m.base_model.base.children())[:24]:
            for p in layer.parameters():
                p.requires_grad = False
    return m.cuda()


def _grads(model):
    return {k: p.grad for k, p in model.named_parameters() if p.requires_grad}


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["tc", "simt"])
def test_embednetpca_step_vs_reference_golden(eng, mode):
    """One triplet step of the engine's EmbedNetPCA (conv5 + NetVLAD + PCA trainable) against the reference on CPU."""
    eng.set_gemm_mode(_modes()[mode])
    eng.conv_mode = _modes()[mode]
    x, sd = golden_inputs()
    model = _model(sd, K, PCA_DIM).train()
    out = model(x.view(-1, 3, H, W).cuda())
    loss = triplet_loss(out, B, 2 + NEG)
    loss.backward()
    grads = {k: v.cpu() for k, v in _grads(model).items()}
    assert set(grads) == set(conv5_and_head())
    # fp32 CUDA cores measure <= 6e-5; on the tensor cores the bf16x3 trunk and NetVLAD differ from the fp32 reference
    # by up to 2.3e-3 in the conv5 gradients (the trainer tests allow 2e-2 there for the same reason)
    errs = check_against_golden(loss.item(), out.detach().cpu(), grads, 1e-4 if mode == "simt" else 1e-2)
    print(mode, errs)


@pytest.mark.gpu
def test_hub_shaped_model_all_layers_trainable_vs_fp64(eng):
    """The hub model's shape (64 clusters, 32768 -> 4096 PCA) with every layer trainable: one step against the fp64
    restatement on the GPU."""
    eng.set_gemm_mode(_modes()["tc"])
    eng.conv_mode = _modes()["tc"]
    sd = synth.make_state_dict(seed=31, sharp=True, with_pca=True, bias_scale=0.02)
    easy, _ = synth.make_sfrs_tuples(seed=32, tuples=1, neg_num=2, n_diff=1, height=64, width=96)
    x = easy.view(-1, 3, 64, 96)
    model = _model(sd, 64, 4096, freeze_below_conv5=False).train()
    out = model(x.cuda())
    loss = triplet_loss(out, 1, 4)
    loss.backward()
    keys = list(sd.keys())
    ref_loss, ref_out, ref = pca_train_step(sd, x, 1, 4, keys, device="cuda")
    got = dict(model.named_parameters())
    errs = {k: rel_l2(got[k].grad.cpu(), ref[k].cpu()) for k in keys}
    errs["out"] = rel_l2(out.detach().cpu(), ref_out.cpu())
    errs["loss"] = abs(loss.item() - ref_loss.item()) / abs(ref_loss.item())
    print({k: f"{v:.2e}" for k, v in errs.items()})
    head = ("pca_layer.weight", "pca_layer.bias", "net_vlad.conv.weight", "net_vlad.centroids", "out", "loss")
    # measured: head <= 3.2e-4, conv5 3e-4, conv1..conv4 up to 7.4e-3 (fp32 ReLU masks of the deep backward flip
    # against fp64 where a pre-activation is within rounding of zero, see test_gpu_train.py)
    assert all(errs[k] < 1e-3 for k in head), errs
    assert all(v < 2e-2 for v in errs.values()), errs


@pytest.mark.gpu
def test_frozen_pca_layer_and_frozen_trunk(eng):
    """requires_grad=False parameters get no .grad: a frozen PCA layer still passes gradients to NetVLAD and conv5; a
    frozen trunk + NetVLAD still trains the PCA layer, with the gradients of the full step."""
    eng.set_gemm_mode(_modes()["tc"])
    eng.conv_mode = _modes()["tc"]
    x, sd = golden_inputs()
    xs = x.view(-1, 3, H, W).cuda()
    full = _model(sd, K, PCA_DIM).train()
    triplet_loss(full(xs), B, 2 + NEG).backward()
    ref = _grads(full)

    m = _model(sd, K, PCA_DIM).train()
    m.pca_layer.weight.requires_grad = False
    m.pca_layer.bias.requires_grad = False
    triplet_loss(m(xs), B, 2 + NEG).backward()
    assert m.pca_layer.weight.grad is None and m.pca_layer.bias.grad is None
    for k, p in m.named_parameters():
        if p.requires_grad:
            assert rel_l2(p.grad.cpu(), ref[k].cpu()) < 1e-5, k

    m = _model(sd, K, PCA_DIM).train()
    for p in list(m.base_model.parameters()) + list(m.net_vlad.parameters()):
        p.requires_grad = False
    triplet_loss(m(xs), B, 2 + NEG).backward()
    assert all(p.grad is None for p in list(m.base_model.parameters()) + list(m.net_vlad.parameters()))
    assert rel_l2(m.pca_layer.weight.grad.cpu(), ref["pca_layer.weight"].cpu()) < 1e-5
    assert rel_l2(m.pca_layer.bias.grad.cpu(), ref["pca_layer.bias"].cpu()) < 1e-5


@pytest.mark.gpu
def test_sgd_steps_lower_the_loss_and_eval_serves_new_weights(eng):
    """Eval outputs are unchanged by a training forward that is not followed by a step (bit for bit), a few SGD
    steps lower the triplet loss, and model.eval() then serves the updated weights."""
    eng.set_gemm_mode(_modes()["tc"])
    eng.conv_mode = _modes()["tc"]
    x, sd = golden_inputs()
    xs = x.view(-1, 3, H, W).cuda()
    model = _model(sd, K, PCA_DIM)
    with torch.no_grad():
        before = model.eval()(xs)
    model.train()
    triplet_loss(model(xs), B, 2 + NEG)
    with torch.no_grad():
        again = model.eval()(xs)
    assert torch.equal(before, again)
    opt = torch.optim.SGD([p for p in model.parameters() if p.requires_grad], lr=0.01)
    model.train()
    losses = []
    for _ in range(5):
        loss = triplet_loss(model(xs), B, 2 + NEG)
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    print(losses)
    assert losses[-1] < losses[0]
    model.eval()
    with torch.no_grad():
        after = model(xs)
    new_sd = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    from oracle import ibl_oracle as O
    want = O.embednetpca_forward(x.view(-1, 3, H, W).double(), {k: v.double() for k, v in new_sd.items()})
    assert rel_l2(after.cpu(), want) < 1e-4
    assert not torch.equal(after, before)


# ---- SASS of the new product kernels (no GPU needed) -------------------------------------------------------------------
def test_pca_backward_kernels_are_wgmma_tma_code():
    """The PCA dgrad / wgrad kernels carry HGMMA and UTMALDG and none of the per-instruction issue loops ptxas builds
    around TMA instructions that are not behind elect.sync (as tests/test_sass_cpu.py checks for the other kernels)."""
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe) or not os.path.exists(LIB):
        pytest.skip("cuobjdump or the built library is missing")
    out = subprocess.run([exe, "-sass", LIB], capture_output=True, text=True, timeout=600).stdout
    counts, fn = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            counts.setdefault(fn, {})
            continue
        if fn is None:
            continue
        for op in ("HGMMA", "UTMALDG", "R2UR.BROADCAST", "BRA.U.ANY"):
            if re.search(r"\b" + re.escape(op), line):
                counts[fn][op] = counts[fn].get(op, 0) + 1
    variants = {k: c for k, c in counts.items() if "pca_bwd_tc_kernel" in k}
    assert len(variants) == 4, sorted(variants)         # dgrad at 32 / 64 / 128 batch rows, wgrad
    for k, c in variants.items():
        assert c.get("HGMMA", 0) > 0 and c.get("UTMALDG", 0) > 0, (k, c)
        assert c.get("BRA.U.ANY", 0) == 0 and c.get("R2UR.BROADCAST", 0) <= 1, (k, c)

"""SURVEY 8 row f1 / BASELINE configs[4]: the training surface -- conv dgrad / wgrad on the tensor cores, pool backward, the
VGG trunk autograd Function, and one SFRS step (trainers.py:235-259) against the UNMODIFIED reference run on CPU
(tests/golden/sfrs_step.npz, oracle/gen_golden_sfrs.py).  Tolerances are stated next to each check."""
import numpy as np
import pytest
import torch

from conftest import load_golden, rel_l2
from openibl_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from openibl_b200.engine import Engine
    return Engine.get(0)


def _bind_vgg(eng, seed=3, bias_scale=0.05):
    sd = synth.make_vgg_weights(seed, bias_scale)
    slots = synth.VGG16_CONV_SLOTS
    ws = [sd[f"base.{s}.weight"].cuda() for s in slots]
    bs = [sd[f"base.{s}.bias"].cuda() for s in slots]
    eng.set_vgg16(ws, bs, force=True)
    return ws, bs


LAYER_CASES = [
    # layer, N, H, W
    (12, 3, 15, 20),     # conv5_3 (no ReLU) on quarter-region sized maps
    (11, 2, 30, 40),     # conv5_2 at the full 480x640 feature size
    (10, 5, 7, 9),       # conv5_1, ragged: partial 16x4 boxes on both axes
    (7, 1, 16, 24),      # conv4_1: 256 -> 512 (Cin tile 128 x 2, Cout tile 128 x 4)
    (2, 1, 20, 33),      # conv2_1: 64 -> 128 (a zero-filled half of the Cin tile)
    (1, 2, 12, 18),      # conv1_2: 64 -> 64
]


@pytest.mark.parametrize("case", LAYER_CASES)
def test_conv_layer_forward_backward_vs_fp64_autograd(eng, case):
    """y = [ReLU](conv(x)+b), dL/dx (tensor-core dgrad = forward kernel on rotated filters), dL/dW (tensor-core wgrad with
    pixel-major operands), dL/db against torch autograd in fp64.  rel-L2 <= 1e-4 (north-star tolerance; bf16x3
    measures ~2e-5)."""
    layer, N, H, W = case
    ws, bs = _bind_vgg(eng)
    w, b = ws[layer], bs[layer]
    cout, cin = w.shape[:2]
    relu = layer != 12
    g = torch.Generator().manual_seed(100 + layer)
    x = torch.randn(N, cin, H, W, generator=g).relu()
    gy = torch.randn(N, cout, H, W, generator=g)
    xd = x.double().requires_grad_(True)
    wd, bd = w.cpu().double().requires_grad_(True), b.cpu().double().requires_grad_(True)
    pre = torch.nn.functional.conv2d(xd, wd, bd, padding=1)
    x_nhwc = x.permute(0, 2, 3, 1).contiguous().cuda()
    y = eng.vgg16_layer_forward(layer, x_nhwc, cout)
    assert rel_l2(y.permute(0, 3, 1, 2).cpu(), pre.detach().relu() if relu else pre.detach()) < 2e-5
    # The ReLU mask of the reference gradient is taken from the ENGINE's forward output: where a pre-activation is
    # within fp32 noise of zero (about 1e-5 of all elements) the fp64 and fp32 forwards disagree on its sign, and one
    # flipped element switches a whole gradient path on or off (rel-L2 ~ sqrt(1e-5) = 3e-3) -- that is a property of
    # ReLU, not of the backward kernels, which must be consistent with the forward they belong to.
    mask = (y.permute(0, 3, 1, 2).cpu() > 0).double() if relu else torch.ones_like(pre)
    (pre * mask * gy.double()).sum().backward()
    gx, gw, gb = eng.vgg16_layer_backward(layer, x_nhwc, y if relu else None, gy.permute(0, 2, 3, 1).contiguous().cuda(),
                                          tuple(w.shape), need_gx=True)
    torch.cuda.synchronize()
    assert rel_l2(gx.permute(0, 3, 1, 2).cpu(), xd.grad) < 1e-4, rel_l2(gx.permute(0, 3, 1, 2).cpu(), xd.grad)
    assert rel_l2(gw.cpu(), wd.grad) < 1e-4, rel_l2(gw.cpu(), wd.grad)
    assert rel_l2(gb.cpu(), bd.grad) < 1e-4, rel_l2(gb.cpu(), bd.grad)


def test_conv1_1_backward_and_pool_backward(eng):
    ws, bs = _bind_vgg(eng)
    g = torch.Generator().manual_seed(9)
    x = torch.randn(2, 3, 20, 28, generator=g)
    gy = torch.randn(2, 64, 20, 28, generator=g)
    xd = x.double()
    wd, bd = ws[0].cpu().double().requires_grad_(True), bs[0].cpu().double().requires_grad_(True)
    yd = torch.nn.functional.conv2d(xd, wd, bd, padding=1).relu()
    (yd * gy.double()).sum().backward()
    y = eng.vgg16_layer_forward(0, x.cuda(), 64)
    assert rel_l2(y.permute(0, 3, 1, 2).cpu(), yd.detach()) < 5e-6
    _, gw, gb = eng.vgg16_layer_backward(0, x.cuda(), y, gy.permute(0, 2, 3, 1).contiguous().cuda(), (64, 3, 3, 3), need_gx=False)
    assert rel_l2(gw.cpu(), wd.grad) < 1e-4 and rel_l2(gb.cpu(), bd.grad) < 1e-4
    # 2x2 max-pool: forward and backward (gradient to the first maximum, as ATen), odd sizes floor
    for (N, H, W, C) in ((2, 9, 14, 64), (1, 6, 6, 8)):
        a = torch.randn(N, C, H, W, generator=g)
        a[:, :, :2, :2] = 1.5                                   # a window of ties
        ad = a.clone().requires_grad_(True)
        p = torch.nn.functional.max_pool2d(ad, 2, 2)
        gp = torch.randn(p.shape, generator=g)
        (p * gp).sum().backward()
        a_nhwc = a.permute(0, 2, 3, 1).contiguous().cuda()
        got = eng.maxpool2x2(a_nhwc)
        assert torch.equal(got.permute(0, 3, 1, 2).cpu(), p.detach())
        gx = eng.maxpool2x2_backward(a_nhwc, gp.permute(0, 2, 3, 1).contiguous().cuda())
        assert torch.equal(gx.permute(0, 3, 1, 2).cpu(), ad.grad)


@pytest.mark.parametrize("n_layers", [1, 2, 4])
def test_vgg16_prefix_forward_vs_fp64(eng, n_layers):
    """The frozen trunk prefix (train_layers='conv2' freezes layers [0, 2)) on an odd input, tensor-core mode, against
    fp64 conv/ReLU/pool; rel-L2 <= 2e-5 as the per-layer tests.  1: the CUDA-core fp32 conv1_1.  2: the separate
    tensor-core conv1_1 and the BN=64 conv1_2 with the fp32 epilogue and fused pool.  4: the fused conv1 kernel
    feeding conv2_x with an fp32 output."""
    from openibl_b200.engine import CONV_TC_BF16X3
    ws, bs = _bind_vgg(eng)
    x = torch.randn(2, 3, 70, 90, generator=torch.Generator().manual_seed(21))
    ref = x.double()
    for item in synth.VGG16_PLAN[: {1: 1, 2: 3, 4: 6}[n_layers]]:
        if item == "P":
            ref = torch.nn.functional.max_pool2d(ref, 2, 2)
        else:
            i = synth.VGG16_CONV_SLOTS.index(item[0])
            ref = torch.nn.functional.conv2d(ref, ws[i].cpu().double(), bs[i].cpu().double(), padding=1).relu()
    mode = eng.conv_mode
    eng.conv_mode = CONV_TC_BF16X3
    try:
        y = eng.vgg16_prefix_forward(x.cuda(), n_layers)
    finally:
        eng.conv_mode = mode
    assert y.shape == ref.permute(0, 2, 3, 1).shape
    err = rel_l2(y.permute(0, 3, 1, 2).cpu(), ref)
    assert err < 2e-5, err


def _freeze_below_conv5(model):
    for layer in list(model.base_model.base.children())[:24]:
        for p in layer.parameters():
            p.requires_grad = False


def _build(seed, tuple_size):
    from ibl import models
    sd = synth.make_state_dict(seed=seed, sharp=True, with_pca=False, bias_scale=0.02)
    m = models.create("embedregionnet", models.create("vgg16", pretrained=False), models.create("netvlad", dim=512),
                      tuple_size=tuple_size)
    m.load_state_dict(sd)
    _freeze_below_conv5(m)
    return m.cuda().train()


@pytest.mark.parametrize("gen", [0, 1])
def test_sfrs_step_losses_and_gradients_vs_reference_golden(eng, gen):
    """One SFRS step, tuple_size 2 (the reference itself can only run tuple_size 1 on torch 2.x; its B = 2 result is
    the mean of two single-tuple runs): losses within 2e-4 relative of the unmodified reference on CPU; gradients:
    NetVLAD parameters within 3e-3 relative L2, conv5 weights within 2e-2 and cosine > 0.9998 -- two ReLUs sit
    between conv5_1 and the loss, and the ~1e-5 of activations whose pre-activation is within fp32 noise of zero take
    a different side of the ReLU in the two implementations (each flip switches a gradient path; measured 8e-3)."""
    from ibl.trainers import SFRSTrainer
    g = load_golden("sfrs_step")
    B, NEG, NDIFF, H, W = 2, 2, 2, 64, 96
    easy, diff = synth.make_sfrs_tuples(seed=31, tuples=B, neg_num=NEG, n_diff=NDIFF, height=H, width=W)
    model, cache = _build(13, B), _build(23, B)
    tr = SFRSTrainer(model, cache, margin=0.1, neg_num=NEG, gpu=0, temp=[0.07, 0.07])
    lh, ls = tr._forward(easy.cuda(), diff.cuda(), "sare_ind", gen)
    assert abs(lh.item() - float(g[f"g{gen}_loss_hard"])) < 2e-4 * max(1.0, abs(float(g[f"g{gen}_loss_hard"])))
    assert abs(ls.item() - float(g[f"g{gen}_loss_soft"])) < 2e-4 * max(1.0, abs(float(g[f"g{gen}_loss_soft"])))
    (lh + 0.5 * ls).backward()
    base = model.base_model.base
    assert base[21].weight.grad is None                      # frozen below conv5
    for slot in (24, 26, 28):
        gw = base[slot].weight.grad.cpu()
        sub, want = gw[::8, ::8].double().flatten(), torch.from_numpy(g[f"g{gen}_w{slot}"]).double().flatten()
        assert rel_l2(sub, want) < 2e-2, (slot, rel_l2(sub, want))
        assert float(sub @ want / (sub.norm() * want.norm())) > 0.9998, slot
        assert abs(float(gw.double().norm()) - float(g[f"g{gen}_w{slot}_norm"])) < 1e-2 * float(g[f"g{gen}_w{slot}_norm"])
        assert rel_l2(base[slot].bias.grad.cpu(), g[f"g{gen}_b{slot}"]) < 2e-2, slot
    assert rel_l2(model.net_vlad.centroids.grad.cpu()[:, ::4], g[f"g{gen}_centroids"]) < 3e-3
    assert rel_l2(model.net_vlad.conv.weight.grad.cpu()[:, ::4, 0, 0], g[f"g{gen}_conv_w"]) < 3e-3


def test_embednet_training_forward_is_differentiable_and_matches_eval(eng):
    """netvlad_img.py trains EmbedNet: the train-mode forward (autograd Functions) equals the eval-mode forward and
    sends gradients to the trainable suffix only."""
    from ibl import models
    sd = synth.make_state_dict(seed=4, sharp=True, with_pca=False, bias_scale=0.02)
    m = models.create("embednet", models.create("vgg16", pretrained=False), models.create("netvlad", dim=512))
    m.load_state_dict(sd)
    _freeze_below_conv5(m)
    m = m.cuda()
    x = synth.make_smooth_images(seed=8, batch=3, height=64, width=96).cuda()
    m.eval()
    with torch.no_grad():
        _, want = m(x)
    m.train()
    pool_x, got = m(x)
    assert got.requires_grad and rel_l2(got.detach().cpu(), want.cpu()) < 2e-5
    got.square().sum().backward()
    assert m.base_model.base[28].weight.grad is not None and m.base_model.base[0].weight.grad is None
    assert torch.isfinite(m.net_vlad.centroids.grad).all()

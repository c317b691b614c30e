"""The backward of the VGG16 trunk for every `train_layers` setting, against float64 references.

1. Every conv layer alone, forward and backward, on ragged maps (H not a multiple of the 4-row box, W not a multiple
   of the 16-column box, W < 16, H < 4, N = 1) and at pixel counts on both sides of the bias-gradient and conv1_1
   wgrad part counts.
2. A long-reduction probe of the tensor-core wgrad: with x >= 0 and dY >= 0 every dW entry is a sum of positive
   products, so an accumulator that loses a little on every addition shows up as a uniform scale below 1.  The
   reference is 9 shifted float64 GEMMs on the device (exact, and independent of cuDNN).
3. The whole trunk through `_VGGTrunkFunction` for conv5 / conv4 / conv3 / conv2 / full, against the float64
   linearisation along the engine's own ReLU masks and pooling argmaxes.  The feature is held to 2e-5 behind the
   CUDA-core forward; behind the tensor-core forward to 1.5e-4 with at most 5e-5 that is not one uniform scale.
4. NetVLAD backward at the SFRS training shape (S = 30 x 40 = 1200 per image, 12 and 48 images) and the 2x2 max-pool
   bit-exact against ATen on a tensor larger than the pool kernels' grid-stride cap.

Every reference is plain float64 torch.  Errors are relative L2 and are printed per case (run with -s)."""
import math

import pytest
import torch
import torch.nn.functional as F

from openibl_b200 import synth

pytestmark = pytest.mark.gpu

POOL_AFTER = {1, 3, 6, 9}                       # conv1_2, conv2_2, conv3_3, conv4_3 feed a 2x2 max-pool
FIRST_TRAINABLE = {"conv5": 10, "conv4": 7, "conv3": 4, "conv2": 2, "full": 0}


@pytest.fixture(scope="module")
def eng():
    from openibl_b200.engine import Engine, CONV_TC_BF16X3
    e = Engine.get(0)
    mode = e.conv_mode
    e.conv_mode = CONV_TC_BF16X3
    yield e
    e.conv_mode = mode


def rel(a, b):
    a, b = a.detach().double(), b.detach().double().to(a.device)
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def scale_bias(got, ref):
    """1 - <got, ref> / <ref, ref>: the part of the error that is one uniform scale (> 0: got is too small)."""
    got, ref = got.detach().double(), ref.detach().double().to(got.device)
    return 1.0 - float((got * ref).sum() / (ref * ref).sum())


def descaled_rel(got, ref):
    """rel-L2 after the best-fit scalar: the error that a uniform scale cannot explain."""
    got, ref = got.detach().double(), ref.detach().double().to(got.device)
    return rel(got * ((got * ref).sum() / (got * got).sum()), ref)


def _bind_vgg(eng, seed=3, bias_scale=0.05):
    sd = synth.make_vgg_weights(seed, bias_scale)
    slots = synth.VGG16_CONV_SLOTS
    ws = [sd[f"base.{s}.weight"].cuda() for s in slots]
    bs = [sd[f"base.{s}.bias"].cuda() for s in slots]
    eng.set_vgg16(ws, bs, force=True)
    return ws, bs


# ---- 1. every layer, forward and backward ---------------------------------------------------------------------------
LAYER_SHAPES = [
    # N, H, W
    (1, 13, 21),      # N = 1; partial 16 x 4 boxes on both axes
    (3, 3, 9),        # H < 4, W < 16; P = 81 < 256: one bias-gradient part per pixel
    (2, 9, 6),        # W < 16 with several box rows
    (4, 45, 70),      # P = 12600 >> 256 bias-gradient parts
]


def _layer_check(eng, layer, N, H, W, seed):
    ws, bs = _bind_vgg(eng)
    w, b = ws[layer], bs[layer]
    cout, cin = w.shape[:2]
    relu = layer != 12
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(N, cin, H, W, device="cuda", generator=g)
    if layer:
        x = x.relu()                             # layers >= 1 see post-ReLU (or pooled post-ReLU) activations
    gy = torch.randn(N, cout, H, W, device="cuda", generator=g)
    xd = x.double().requires_grad_(layer > 0)
    wd, bd = w.double().requires_grad_(True), b.double().requires_grad_(True)
    pre = F.conv2d(xd, wd, bd, padding=1)
    x_in = x.contiguous() if layer == 0 else x.permute(0, 2, 3, 1).contiguous()
    y = eng.vgg16_layer_forward(layer, x_in, cout)
    y_nchw = y.permute(0, 3, 1, 2)
    err_y = rel(y_nchw, pre.relu() if relu else pre)
    # the reference's ReLU mask is the ENGINE's: where a pre-activation is within fp32 noise of zero the two forwards
    # may disagree on its sign, and one flip switches a whole gradient path -- a property of ReLU, not of the backward
    mask = (y_nchw > 0).double() if relu else torch.ones_like(pre)
    (pre * mask * gy.double()).sum().backward()
    gx, gw, gb = eng.vgg16_layer_backward(layer, x_in, y if relu else None, gy.permute(0, 2, 3, 1).contiguous(),
                                          tuple(w.shape), need_gx=layer > 0)
    torch.cuda.synchronize()
    err_gx = rel(gx.permute(0, 3, 1, 2), xd.grad) if layer else 0.0
    err_gw, err_gb = rel(gw, wd.grad), rel(gb, bd.grad)
    print(f"\nlayer {layer:2d} N={N} H={H} W={W}: y {err_y:.2e}  gx {err_gx:.2e}  gW {err_gw:.2e}  gb {err_gb:.2e}")
    assert err_y <= 2e-5, err_y
    assert err_gx <= 1e-4, err_gx
    assert err_gw <= 1e-4, err_gw
    assert err_gb <= 1e-4, err_gb


@pytest.mark.parametrize("shape", LAYER_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("layer", range(13))
def test_layer_forward_backward_vs_fp64(eng, layer, shape):
    _layer_check(eng, layer, *shape, seed=1000 + 13 * LAYER_SHAPES.index(shape) + layer)


def test_conv1_1_wgrad_millions_of_pixels(eng):
    """conv1_1's CUDA-core wgrad splits the N*H*W pixels into 1024 equal chunks: at 7 x 479 x 641 a chunk is 2099
    pixels, which does not divide the 307039 pixels of an image, so chunks straddle image boundaries."""
    N, H, W = 7, 479, 641
    assert (H * W) % math.ceil(N * H * W / 1024) != 0
    _layer_check(eng, 0, N, H, W, seed=77)


# ---- 2. long-reduction probe of the tensor-core wgrad ---------------------------------------------------------------
PROBE_CASES = [
    # layer, N, H, W, 64-pixel boxes per split on a 132-SM H100
    (1, 1, 40, 48, 1),           # conv1_2 (64 -> 64, 9 CTAs per split)
    (1, 2, 80, 192, 16),
    (1, 4, 480, 256, 256),
    (1, 12, 480, 640, 1920),     # conv1_2 under --layers full, 12 images (tuple_size 1) at 480 x 640
    (1, 48, 480, 640, 7680),     # the same with tuple_size 4
    (11, 1, 4, 32, 1),           # conv5_2 (512 -> 512, 144 CTAs per split)
    (11, 1, 32, 64, 16),
    (11, 2, 64, 256, 256),
    (11, 12, 30, 40, 144),       # conv5, tuple_size 1
    (11, 48, 30, 40, 576),       # conv5, tuple_size 4
]


def _boxes_per_split(N, H, W, cin, cout, sms):
    items = 9 * math.ceil(cout / 128) * math.ceil(cin / 128)
    boxes = N * math.ceil(H / 4) * math.ceil(W / 16)
    splits = max(1, min(math.ceil(2 * sms / items), boxes, 64))
    return math.ceil(boxes / splits)


def _wgrad_fp64(x, gy, chunk):
    """dW[co,ci,kh,kw] = sum_{n,h,w} gy[n,h,w,co] x[n,h+kh-1,w+kw-1,ci] (NHWC inputs, zero padding), in float64 as
    9 shifted GEMMs per chunk of images; also db[co] = sum gy."""
    N, H, W, ci = x.shape
    co = gy.shape[3]
    dw = torch.zeros(co, ci, 3, 3, dtype=torch.float64, device=x.device)
    db = torch.zeros(co, dtype=torch.float64, device=x.device)
    for n0 in range(0, N, chunk):
        xs = F.pad(x[n0:n0 + chunk].double(), (0, 0, 1, 1, 1, 1))
        g = gy[n0:n0 + chunk].double().reshape(-1, co)
        db += g.sum(0)
        for kh in range(3):
            for kw in range(3):
                dw[:, :, kh, kw] += g.t() @ xs[:, kh:kh + H, kw:kw + W, :].reshape(-1, ci)
        del xs, g
    return dw, db


def _probe(eng, layer, N, H, W, signed):
    ws, _ = _bind_vgg(eng)
    cout, cin = ws[layer].shape[:2]
    assert cin == cout                             # the input doubles as the (all-positive) ReLU output below
    g = torch.Generator(device="cuda").manual_seed(500 + layer + N)
    x = torch.randn(N, H, W, cin, device="cuda", generator=g).abs_()
    gy = torch.randn(N, H, W, cout, device="cuda", generator=g)
    if not signed:
        gy.abs_()
    # y = x: the layer's ReLU mask keeps every pixel where x > 0 (the reference applies the same mask)
    _, gw, gb = eng.vgg16_layer_backward(layer, x, x, gy, tuple(ws[layer].shape), need_gx=False)
    _, gw2, gb2 = eng.vgg16_layer_backward(layer, x, x, gy, tuple(ws[layer].shape), need_gx=False)
    assert torch.equal(gw, gw2) and torch.equal(gb, gb2)          # a fixed summation order: bit-identical reruns
    del gw2, gb2
    gy.mul_(x > 0)
    ref_w, ref_b = _wgrad_fp64(x, gy, chunk=max(1, (1 << 26) // (H * W * max(cin, cout))))
    del x, gy
    return rel(gw, ref_w), rel(gb, ref_b), scale_bias(gw, ref_w)


@pytest.mark.parametrize("case", PROBE_CASES, ids=lambda c: f"L{c[0]}-{c[1]}x{c[2]}x{c[3]}-{c[4]}boxes")
def test_wgrad_long_reduction_has_no_scale_bias(eng, case):
    """|bias| <= 1e-5 with bias = 1 - <got, ref> / <ref, ref>.  bf16x3 operand rounding is unbiased and averages far
    below 1e-5 over these sums of thousands of positive products, so a failure is a biased accumulation."""
    layer, N, H, W, per_split = case
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    got_per_split = _boxes_per_split(N, H, W, 64 if layer == 1 else 512, 64 if layer == 1 else 512, sms)
    if sms == 132:
        assert got_per_split == per_split
    err_w, err_b, bias = _probe(eng, layer, N, H, W, signed=False)
    torch.cuda.empty_cache()
    print(f"\nwgrad probe layer {layer} N={N} H={H} W={W} ({got_per_split} boxes/split, "
          f"{12 * got_per_split} accumulations/chain): gW {err_w:.2e}  scale bias {bias:+.2e}  gb {err_b:.2e}")
    assert err_w <= 1e-4, err_w
    assert abs(bias) <= 1e-5, bias
    assert err_b <= 1e-4, err_b


def test_wgrad_longest_reduction_signed(eng):
    """Random-sign dY at the longest conv1_2 chain (48 x 480 x 640): cancellation instead of a pure scale."""
    err_w, err_b, bias = _probe(eng, 1, 48, 480, 640, signed=True)
    torch.cuda.empty_cache()
    print(f"\nwgrad signed layer 1 N=48 H=480 W=640: gW {err_w:.2e}  gb {err_b:.2e}")
    assert err_w <= 1e-4, err_w
    assert err_b <= 1e-4, err_b


# ---- 3. the whole trunk ---------------------------------------------------------------------------------------------
def _window_argmax(t):
    """[N,C,H,W] -> [N,C,H//2,W//2] index 0..3 of the FIRST maximum of each 2x2 window in row-major order (as ATen);
    floor pooling drops a trailing odd row / column."""
    return _windows(t).argmax(-1)


def _windows(t):
    N, C, H, W = t.shape
    oh, ow = H // 2, W // 2
    return t[:, :, :2 * oh, :2 * ow].reshape(N, C, oh, 2, ow, 2).permute(0, 1, 2, 4, 3, 5).reshape(N, C, oh, ow, 4)


def _take(t, k):
    return _windows(t).gather(-1, k.unsqueeze(-1)).squeeze(-1)


def _choice_disagreements(x, ws, bs, saved, first):
    """The float64 network's own ReLU masks and argmaxes, from the image, against the engine's (layers >= first).
    Returns (disagreements, elements compared, largest float64 margin of a disagreement in units of the rms
    difference between the engine's and the float64 activations of that layer)."""
    bad, total, worst = 0, 0, 0.0
    h = x.double()
    for l in range(13):
        pre = F.conv2d(h, ws[l].detach().double(), bs[l].detach().double(), padding=1)
        y = pre.relu() if l != 12 else pre
        if l >= first:
            y_e = saved[2 * (l - first) + 1].permute(0, 3, 1, 2)
            noise = float((y_e.double() - y).norm()) / math.sqrt(y.numel())
            if l != 12:
                dis = (y_e > 0) != (pre > 0)
                bad, total = bad + int(dis.sum()), total + pre.numel()
                if dis.any():
                    worst = max(worst, float(pre[dis].abs().max()) / noise)
            if l in POOL_AFTER:
                k_own, k_e = _window_argmax(y), _window_argmax(y_e)
                dis = k_own != k_e
                bad, total = bad + int(dis.sum()), total + dis.numel()
                if dis.any():
                    margin = (_take(y, k_own) - _take(y, k_e))[dis]
                    worst = max(worst, float(margin.max()) / noise)
        h = _take(y, _window_argmax(y)) if l in POOL_AFTER else y
    return bad, total, worst


def _trunk_check(eng, train_layers, mode, N, H, W, seed):
    from ibl import models
    from openibl_b200.engine import CONV_SIMT_FP32, CONV_TC_BF16X3
    m = models.create("vgg16", pretrained=False)
    m.load_state_dict(synth.make_vgg_weights(seed, bias_scale=0.05))
    for layer in list(m.base.children())[: m._fix_layers[train_layers]]:
        for p in layer.parameters():
            p.requires_grad = False
    m = m.cuda().train()
    first = FIRST_TRAINABLE[train_layers]
    assert m.first_trainable_layer() == first
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(N, 3, H, W, device="cuda", generator=g)
    eng.conv_mode = {"simt": CONV_SIMT_FP32, "tc": CONV_TC_BF16X3}[mode]
    try:
        _, feat = m(x)
    finally:
        eng.conv_mode = CONV_TC_BF16X3
    # (input, post-ReLU pre-pool output) of every trainable layer: exactly what the backward reads
    saved = feat.grad_fn.saved_tensors
    assert len(saved) == 2 * (13 - first)
    G = torch.randn(feat.shape, device="cuda", generator=g)
    (feat * G).sum().backward()
    ws, bs = m.conv_params()

    # float64 linearisation along the engine's path: its ReLU masks and its first-maximum argmaxes
    wd = [w.detach().double().requires_grad_(l >= first) for l, w in enumerate(ws)]
    bd = [b.detach().double().requires_grad_(l >= first) for l, b in enumerate(bs)]
    h = saved[0].double() if first == 0 else saved[0].permute(0, 3, 1, 2).double()
    for l in range(first, 13):
        y_e = saved[2 * (l - first) + 1].permute(0, 3, 1, 2)
        pre = F.conv2d(h, wd[l], bd[l], padding=1)
        h = pre * (y_e > 0) if l != 12 else pre
        if l in POOL_AFTER:
            h = _take(h, _window_argmax(y_e))
    err_feat, feat_scale, feat_desc = rel(feat, h), scale_bias(feat, h), descaled_rel(feat, h)
    (h * G.double()).sum().backward()
    errs = []
    for l in range(13):
        if l < first:
            assert ws[l].grad is None and bs[l].grad is None, l
            continue
        errs.append((l, rel(ws[l].grad, wd[l].grad), rel(bs[l].grad, bd[l].grad), scale_bias(ws[l].grad, wd[l].grad),
                     descaled_rel(ws[l].grad, wd[l].grad), descaled_rel(bs[l].grad, bd[l].grad)))
    del h, wd, bd
    with torch.no_grad():
        bad, total, worst = _choice_disagreements(x, ws, bs, saved, first)
    print(f"\ntrunk {train_layers} ({mode}) {N}x3x{H}x{W}: feat {err_feat:.2e} (scale {feat_scale:+.2e}, descaled "
          f"{feat_desc:.2e})  mask/argmax disagreements {bad}/{total} (largest margin {worst:.2f} x noise)")
    for l, ew, eb, sw, dw, db in errs:
        print(f"  layer {l:2d}: gW {ew:.2e} (scale {sw:+.2e}, descaled {dw:.2e})  gb {eb:.2e} (descaled {db:.2e})")
    if mode == "simt":
        assert err_feat <= 2e-5, err_feat
    else:
        # the tensor-core forward shrinks every layer's output by up to ~1.4e-5 (its fp32 accumulator rounds toward
        # zero over the 864 MMAs of a 512-channel layer; DESIGN 3), which adds up over the trunk to one uniform scale
        # of ~9e-5 that the L2 normalisations after the trunk cancel; what a scale cannot explain stays small
        assert err_feat <= 1.5e-4, err_feat
        assert feat_desc <= 5e-5, feat_desc
    for l, ew, eb, sw, dw, db in errs:
        # the same scale enters the gradients through dgrad (the forward kernel on dY), layer by layer
        assert ew <= 1e-4, (l, ew)
        assert eb <= 1e-4, (l, eb)
        assert dw <= 4e-5 and db <= 4e-5, (l, dw, db)
    assert bad <= 1e-4 * total, (bad, total)
    assert worst <= 10.0, worst


@pytest.mark.parametrize("mode", ["tc", "simt"])
@pytest.mark.parametrize("train_layers", ["conv5", "conv4", "conv3", "conv2", "full"])
def test_trunk_backward_vs_fp64_linearisation(eng, train_layers, mode):
    """2 x 3 x 70 x 90: floor pooling drops a row or column at 70->35->17->8->4 and 90->45->22->11->5.  In "simt"
    mode the CUDA-core forward feeds the tensor-core backward."""
    _trunk_check(eng, train_layers, mode, 2, 70, 90, seed=41)


def test_trunk_backward_full_480x640(eng):
    _trunk_check(eng, "full", "tc", 2, 480, 640, seed=43)


# ---- 4. NetVLAD backward at the training shape, max-pool bit-exactness ------------------------------------------------
@pytest.mark.parametrize("N", [12, 48])
def test_netvlad_backward_at_training_shape(eng, N):
    """S = 30 x 40 per image as conv5 of a 480 x 640 image; the weight gradient then reduces over N * 1200 rows
    (57,600 at N = 48).  Sharp parameters (alpha ~ 280) as in training; tolerances as the small-shape test."""
    from ibl import models
    from oracle import ibl_oracle as O
    p = synth.make_netvlad_params(seed=4, sharp=True)
    g = torch.Generator(device="cuda").manual_seed(60 + N)
    x = torch.randn(N, 512, 30, 40, device="cuda", generator=g) * 2.0 + 0.3
    G = torch.randn(N, 64, 512, device="cuda", generator=g)
    xd = x.double().requires_grad_(True)
    wd = p["conv_weight"].cuda().double().requires_grad_(True)
    cd = p["centroids"].cuda().double().requires_grad_(True)
    want = O.netvlad(xd, wd, cd)
    (want * G.double()).sum().backward()
    layer = models.create("netvlad", dim=512).cuda().train()
    layer.centroids.data.copy_(p["centroids"])
    layer.conv.weight.data.copy_(p["conv_weight"])
    xg = x.clone().requires_grad_(True)
    out = layer(xg)
    (out * G).sum().backward()
    errs = (rel(out, want), rel(xg.grad, xd.grad), rel(layer.conv.weight.grad, wd.grad), rel(layer.centroids.grad, cd.grad))
    print(f"\nnetvlad N={N} S=1200: out {errs[0]:.2e}  dx {errs[1]:.2e}  dW {errs[2]:.2e}  dC {errs[3]:.2e}")
    assert errs[0] <= 3e-5, errs[0]
    assert max(errs[1:]) <= 3e-4, errs          # sharp softmax amplifies fp32 rounding in dz


def test_maxpool2x2_bit_exact_vs_aten_beyond_grid_stride(eng):
    """C = 512, odd H and W, 3 * 31 * 41 * 512 = 1.95M elements > 132 * 32 blocks * 256 threads, so the pool kernels
    take more than one grid-stride step.  Values on a 0.25 grid give ties everywhere, positive ones included; the
    gradient must go to the first maximum of a window in row-major order, as ATen's."""
    N, H, W, C = 3, 31, 41, 512
    assert N * H * W * C > 132 * 32 * 256
    g = torch.Generator().manual_seed(17)
    a = torch.randint(-4, 5, (N, C, H, W), generator=g).float() * 0.25
    a[:, :, 4:6, 6:8] = 0.75                                        # a whole window of positive ties
    ad = a.clone().requires_grad_(True)
    p = F.max_pool2d(ad, 2, 2)
    gp = torch.randn(p.shape, generator=g)
    (p * gp).sum().backward()
    a_nhwc = a.permute(0, 2, 3, 1).contiguous().cuda()
    got = eng.maxpool2x2(a_nhwc)
    assert torch.equal(got.permute(0, 3, 1, 2).cpu(), p.detach())
    gx = eng.maxpool2x2_backward(a_nhwc, gp.permute(0, 2, 3, 1).contiguous().cuda())
    assert torch.equal(gx.permute(0, 3, 1, 2).cpu(), ad.grad)

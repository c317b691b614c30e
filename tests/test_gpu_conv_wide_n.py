"""The 256-pixel 3x3 conv kernel (64 output channels x 256 pixels per tile, weights in registers, pixels as the wgmma B
operand read through halo views): the register-A MMA on every view start the nine taps use, both patch shapes against
fp64 with ragged borders, pool, both output modes and several tiles per CTA, batch invariance, and the same inputs
through both kernels."""
import pytest
import torch

from conftest import rel_l2

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from openibl_b200.engine import Engine
    return Engine.get(0)


@pytest.mark.parametrize("tw,n", [(32, 64), (16, 128)])
def test_wgmma_rs_halo_views(eng, tw, n):
    """One register-A wgmma against the exact integer product, B read through the halo view of every tap and pixel
    view: 16x16 patches as n128 views with 8-pixel groups 2304 B apart (the kernel's), 8x32 patches as n64 views
    4352 B apart."""
    from openibl_b200._cabi import check
    from openibl_b200.engine import _ptr, _stream
    pitch, hrows = tw + 2, 256 // tw + 2
    g = torch.Generator(device="cuda").manual_seed(tw)
    Wt = torch.randint(-8, 9, (64, 64), device="cuda", generator=g).to(torch.bfloat16)
    X = torch.randint(-8, 9, (hrows * pitch, 64), device="cuda", generator=g).to(torch.bfloat16)
    D = torch.empty(64, n, device="cuda")
    j = torch.arange(n, device="cuda")
    for kh in range(3):
        for kw in range(3):
            for v in range(256 // n):
                s0 = kh * pitch + kw + 8 * v
                want = Wt.float() @ X[s0 + (j // 8) * pitch + j % 8].float().t()
                check(eng.lib.ibl_debug_wgmma_rs_halo_view(eng.h, _ptr(Wt), _ptr(X), pitch, hrows, n, s0, _ptr(D),
                                                           _stream(0)), "probe")
                torch.cuda.synchronize()
                assert torch.equal(D, want), (tw, kh, kw, v)


WIDE_CASES = [
    # N, H, W, cin, cout, relu, pool              patch, tiles (> 132 CTAs: several per CTA)
    (4, 120, 160, 128, 256, True, False),       # ragged height (conv3_x's map), 4 x 80 x 4 = 1280 tiles
    (3, 240, 320, 64, 128, True, True),         # conv2_1's map + pool, 3 x 300 x 2 = 1800 tiles
    (5, 60, 80, 256, 512, True, False),         # ragged height (conv4_x), Cin 256, 5 x 20 x 8 = 800 tiles
    (6, 20, 70, 512, 64, False, False),         # ragged on both axes, Cin 512 (8 chunks), Cout 64: 6 x 10 = 60 tiles
    (16, 44, 36, 128, 192, True, True),         # ragged on both axes + pool, odd Cout / 64, 16 x 9 x 3 = 432 tiles
    (9, 24, 64, 64, 128, False, True),          # ragged height + pool, no ReLU, 9 x 8 x 2 = 144 tiles
]


def _ref(x, w, b, relu, pool):
    ref = torch.nn.functional.conv2d(x.double(), w.double(), b.double(), padding=1)
    if relu:
        ref = ref.relu()
    if pool:
        ref = torch.nn.functional.max_pool2d(ref, 2, 2)
    return ref.permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("case", WIDE_CASES)
def test_wide_conv_vs_fp64(eng, case):
    N, H, W, cin, cout, relu, pool = case
    g = torch.Generator().manual_seed(sum(case[:5]))
    x = torch.randn(N, cin, H, W, generator=g)
    w = torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (cin * 9)) ** 0.5
    b = torch.randn(cout, generator=g) * 0.1
    ref = _ref(x, w, b, relu, pool)
    xd = x.permute(0, 2, 3, 1).contiguous().cuda()
    for name, mode in (("tc-f32", 1), ("tc-planes", 2)):
        y = eng.debug_conv3x3(xd, w.cuda(), b.cuda(), relu=relu, pool=pool, mode=mode, variant=2).cpu()
        assert y.shape == ref.shape, name
        assert rel_l2(y, ref) < 2e-5, (name, rel_l2(y, ref))
        if mode == 2:
            # the last image alone gives the same bits as its slice of the batch
            one = eng.debug_conv3x3(xd[N - 1:].contiguous(), w.cuda(), b.cuda(), relu=relu, pool=pool, mode=mode,
                                    variant=2)
            assert torch.equal(one.cpu(), y[N - 1:]), name


@pytest.mark.parametrize("case", WIDE_CASES[:3])
def test_wide_and_128_pixel_kernels_agree(eng, case):
    """Both halo kernels on the same inputs give the same bits: the same products in the same order per output
    (chunk, tap, k16, then W_hi.X_lo, W_lo.X_hi, W_hi.X_hi), the operand roles swapped.  (Cout = 64 or 192 would put
    the 128-pixel side on the 64-channel kernel, which walks K tap-major.)"""
    N, H, W, cin, cout, relu, pool = case
    g = torch.Generator().manual_seed(7 + sum(case[:5]))
    x = torch.randn(N, H, W, cin, generator=g).cuda()
    w = (torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (cin * 9)) ** 0.5).cuda()
    b = (torch.randn(cout, generator=g) * 0.1).cuda()
    for mode in (1, 2):
        y1 = eng.debug_conv3x3(x, w, b, relu=relu, pool=pool, mode=mode, variant=1)
        y2 = eng.debug_conv3x3(x, w, b, relu=relu, pool=pool, mode=mode, variant=2)
        assert torch.equal(y1, y2), mode


def test_wide_last_layer_norm_partials(eng):
    """conv5_3 on the 256-pixel kernel (a 16x16 map) hands NetVLAD its planes and per-warp |x|^2 partials: the
    descriptors match those of the 128-pixel kernels' per-tile partials."""
    from openibl_b200 import synth
    sd = {k: v.cuda() for k, v in synth.make_state_dict(seed=5, with_pca=True, pca_dim=128, bias_scale=0.05).items()}
    slots = synth.VGG16_CONV_SLOTS
    eng.set_vgg16([sd[f"base_model.base.{s}.weight"] for s in slots], [sd[f"base_model.base.{s}.bias"] for s in slots])
    eng.set_netvlad(sd["net_vlad.conv.weight"], sd["net_vlad.centroids"])
    eng.set_pca(sd["pca_layer.weight"], sd["pca_layer.bias"])
    x = synth.make_images(seed=8, batch=2, height=256, width=256).cuda()
    out = {}
    for variant in (1, 0):
        eng.lib.ibl_debug_set_conv3x3_variant(eng.h, variant)
        try:
            out[variant], _ = eng.extract(x, pca=True)
            torch.cuda.synchronize()
        finally:
            eng.lib.ibl_debug_set_conv3x3_variant(eng.h, 0)
    assert rel_l2(out[0].cpu(), out[1].cpu()) < 1e-6

"""The fused conv1 kernel on 16x16 patches against the unfused path, bit for bit: conv1_1 on its own kernel, then conv1_2
with 2x2 max-pool on the 128-pixel box kernel or the 256-pixel halo kernel, with an fp32 epilogue split into the same
bf16 hi/lo planes.  Both convolutions add their products in the same order in the fused and the unfused kernels, and
max-pooling before bias and ReLU gives the same fp32 values as after (both are monotone), so the planes must be equal.
Inputs have more than 2 x 132 patches (every CTA runs several, both consumer warpgroups alternate), maps ragged on both
axes and odd sizes (floor pooling), one image and batches; every image alone gives the same bits as inside its batch."""
import pytest
import torch

from openibl_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from openibl_b200.engine import Engine
    e = Engine.get(0)
    sd = synth.make_vgg_weights(11, bias_scale=0.05)
    slots = synth.VGG16_CONV_SLOTS
    e.set_vgg16([sd[f"base.{s}.weight"].cuda() for s in slots], [sd[f"base.{s}.bias"].cuda() for s in slots])
    return e


CASES = [
    # N, H, W                  16x16 patches
    (1, 301, 287),           # one image, odd H and W, ragged on both axes: 19 x 18 = 342 patches
    (6, 90, 125),            # a batch, ragged on both axes, odd W: 6 x 6 x 8 = 288 patches
    (24, 45, 62),            # odd H (the last row is pooled away), 24 x 3 x 4 = 288 patches
]


def _unfused(eng, x, variant):
    """conv1_1 -> ReLU -> conv1_2 -> ReLU -> 2x2 max-pool through the unfused kernels, as the fused kernel's planes."""
    from openibl_b200._cabi import check
    check(eng.lib.ibl_debug_set_conv3x3_variant(eng.h, variant), "ibl_debug_set_conv3x3_variant")
    try:
        y = eng.vgg16_prefix_forward(x, 2)       # conv1_2 is the last layer: pooled, fp32 NHWC
    finally:
        eng.lib.ibl_debug_set_conv3x3_variant(eng.h, 0)
    hi = y.to(torch.bfloat16)
    lo = (y - hi.float()).to(torch.bfloat16)
    return hi, lo


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("variant", [1, 2], ids=["box", "wide"])
def test_conv1_fused_equals_unfused(eng, case, variant):
    N, H, W = case
    x = torch.randn(N, 3, H, W, generator=torch.Generator().manual_seed(N * H + W)).cuda()
    hi, lo = eng.debug_conv1_fused(x)
    want_hi, want_lo = _unfused(eng, x, variant)
    torch.cuda.synchronize()
    assert hi.shape == (N, H // 2, W // 2, 64) and want_hi.shape == hi.shape
    assert torch.equal(hi, want_hi) and torch.equal(lo, want_lo)


@pytest.mark.parametrize("case", CASES[1:])
def test_conv1_fused_batch_invariant(eng, case):
    N, H, W = case
    x = torch.randn(N, 3, H, W, generator=torch.Generator().manual_seed(H * W)).cuda()
    hi, lo = eng.debug_conv1_fused(x)
    for i in (0, N // 2, N - 1):
        hi1, lo1 = eng.debug_conv1_fused(x[i:i + 1].contiguous())
        torch.cuda.synchronize()
        assert torch.equal(hi1, hi[i:i + 1]) and torch.equal(lo1, lo[i:i + 1]), i

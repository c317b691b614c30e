"""The fused conv1_1 + ReLU + conv1_2 + ReLU + 2x2 max-pool kernel on its own, against fp64: inputs with several
tiles per CTA (so both consumer warpgroups and the hand-over between them run), ragged and odd maps (floor pooling),
one image and a batch; and every image alone gives the same bits as inside its batch."""
import pytest
import torch

from conftest import rel_l2
from openibl_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from openibl_b200.engine import Engine
    return Engine.get(0)


def _bind(eng):
    sd = synth.make_vgg_weights(7, bias_scale=0.05)
    slots = synth.VGG16_CONV_SLOTS
    ws = [sd[f"base.{s}.weight"] for s in slots]
    bs = [sd[f"base.{s}.bias"] for s in slots]
    eng.set_vgg16([w.cuda() for w in ws], [b.cuda() for b in bs])
    return ws, bs


CASES = [
    # N, H, W                  16x8 tiles (> 2 x 132: every CTA runs several, both consumers alternate)
    (1, 171, 203),           # one image, odd H and W, ragged on both axes: 11 x 26 = 286 tiles
    (6, 62, 90),             # a batch, ragged on both axes: 6 x 4 x 12 = 288 tiles
    (12, 45, 60),            # odd H (the last row is pooled away), W not a multiple of 8: 12 x 3 x 8 = 288 tiles
]


@pytest.mark.parametrize("case", CASES)
def test_conv1_fused_vs_fp64(eng, case):
    N, H, W = case
    ws, bs = _bind(eng)
    x = torch.randn(N, 3, H, W, generator=torch.Generator().manual_seed(N * H + W))
    ref = torch.nn.functional.conv2d(x.double(), ws[0].double(), bs[0].double(), padding=1).relu()
    ref = torch.nn.functional.conv2d(ref, ws[1].double(), bs[1].double(), padding=1).relu()
    ref = torch.nn.functional.max_pool2d(ref, 2, 2).permute(0, 2, 3, 1)
    xd = x.cuda()
    hi, lo = eng.debug_conv1_fused(xd)
    torch.cuda.synchronize()
    assert hi.shape == ref.shape and lo.shape == ref.shape
    y = hi.double().cpu() + lo.double().cpu()
    err = rel_l2(y, ref)
    assert err < 2e-5, err
    # the last image alone (fewer tiles per CTA, another split between the consumers) gives the same bits
    hi1, lo1 = eng.debug_conv1_fused(xd[N - 1:].contiguous())
    torch.cuda.synchronize()
    assert torch.equal(hi1.cpu(), hi[N - 1:].cpu()) and torch.equal(lo1.cpu(), lo[N - 1:].cpu())

"""The halo conv kernel with two consumer warpgroups (ping-pong) and both patch shapes: layers large enough that every
CTA runs several tiles, so both consumers and the hand-over between them are exercised, on maps where the 8x16 and
the 16x8 patch are chosen with ragged borders; and the tensor-core operand view the 8x16 patch reads."""
import pytest
import torch

from conftest import rel_l2

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from openibl_b200.engine import Engine
    return Engine.get(0)


PINGPONG_CASES = [
    # N, H, W, cin, cout, relu, pool              patch chosen, tiles (> 132 CTAs: several per CTA)
    (16, 20, 35, 128, 256, True, False),        # 8x16, ragged on both axes, 3x3 patches x 2 N tiles x 16 = 288
    (16, 20, 35, 128, 128, True, True),         # 8x16 + fused pool, odd width: floor pooling, 144 tiles
    (5, 120, 160, 64, 128, False, False),       # 8x16 tiling 120x160 exactly (conv3_1-like), 750 tiles
    (16, 30, 40, 128, 128, True, True),         # 16x8, ragged height + pool, 160 tiles
    (9, 30, 20, 512, 512, False, False),        # 16x8, ragged on both axes, Cin = 512: 8 chunks per tile, 216 tiles
]


@pytest.mark.parametrize("case", PINGPONG_CASES)
def test_halo_conv_pingpong_vs_fp64(eng, case):
    N, H, W, cin, cout, relu, pool = case
    g = torch.Generator().manual_seed(sum(case[:5]))
    x = torch.randn(N, cin, H, W, generator=g)
    w = torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (cin * 9)) ** 0.5
    b = torch.randn(cout, generator=g) * 0.1
    ref = torch.nn.functional.conv2d(x.double(), w.double(), b.double(), padding=1)
    if relu:
        ref = ref.relu()
    if pool:
        ref = torch.nn.functional.max_pool2d(ref, 2, 2)
    ref = ref.permute(0, 2, 3, 1).contiguous()
    xd = x.permute(0, 2, 3, 1).contiguous().cuda()
    for name, mode in (("tc-f32", 1), ("tc-planes", 2)):
        y = eng.debug_conv3x3(xd, w.cuda(), b.cuda(), relu=relu, pool=pool, mode=mode, bn=128).cpu()
        assert y.shape == ref.shape, name
        assert rel_l2(y, ref) < 2e-5, (name, rel_l2(y, ref))
        # every image on its own (one or two tiles per CTA) gives the same bits as the batch
        if mode == 2:
            one = eng.debug_conv3x3(xd[N - 1:].contiguous(), w.cuda(), b.cuda(), relu=relu, pool=pool, mode=mode, bn=128)
            assert torch.equal(one.cpu(), y[N - 1:]), name


def test_umma_sw128_operand_8x16_halo_view():
    """The 8x16 patch reads its taps out of an 18-pixel-wide halo tile: 8-row groups 18 rows (2304 B) apart and the
    second m64 half (patch columns 8-15) 8 rows after the first."""
    from openibl_b200._cabi import check
    from openibl_b200.engine import Engine, _ptr, _stream
    e = Engine.get(0)
    g = torch.Generator(device="cuda").manual_seed(6)
    rows = 200
    A = torch.randint(-8, 9, (rows, 64), device="cuda", generator=g).to(torch.bfloat16)
    B = torch.randint(-8, 9, (64, 64), device="cuda", generator=g).to(torch.bfloat16)
    D = torch.empty(128, 64, device="cuda")
    m = torch.arange(128, device="cuda")
    for group_rows, half_rows, s0 in ((18, 8, 0), (18, 8, 1), (18, 8, 2), (18, 8, 19), (18, 8, 38), (10, 80, 11)):
        idx = s0 + ((m % 64) // 8) * group_rows + (m // 64) * half_rows + (m % 8)
        want = A[idx].float() @ B.float().t()
        check(e.lib.ibl_debug_umma_halo_view(e.h, _ptr(A), rows, _ptr(B), s0, group_rows, half_rows, _ptr(D),
                                             _stream(0)), "probe")
        torch.cuda.synchronize()
        assert torch.equal(D, want), (group_rows, half_rows, s0)

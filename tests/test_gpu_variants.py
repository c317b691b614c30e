"""Kernel variants that are selected by environment variables (read once per process) are exercised in child
processes, each running the relevant subset of the parity tests: both staging modes and the SM pairs of the tensor-core
conv, the separate conv1_1 / conv1_2 kernels (tensor-core or CUDA-core conv1_1) and the bf16x3 distance screening kernel
on one SM or on SM pairs must give the same answers as the defaults.  Also pins the hardware property halo-staged
convolution relies on."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

VARIANTS = [
    # env, -k expression
    ({"IBL_CONV_HALO": "2"}, "conv3x3 or small or odd"),                    # halo staging on every N tile
    ({"IBL_CONV_HALO": "0", "IBL_CONV_2SM": "0"}, "conv3x3 or small or odd"),   # im2col boxes, one SM per tile
    ({"IBL_CONV_2SM": "2", "IBL_CONV_HALO": "0"}, "conv3x3 or odd"),        # SM pairs on every layer
    ({"IBL_CONV1_FUSED": "0"}, "small or odd or hub or tokyo"),             # separate conv1_1 / conv1_2 kernels
    ({"IBL_CONV1_FUSED": "0", "IBL_CONV1_SIMT": "1"}, "small or odd"),      # ... with the CUDA-core conv1_1
    ({"IBL_DIST_SCREEN": "3"}, "retrieval or topk"),                         # bf16x3 screening (tc_gemm.cu) on SM pairs
    ({"IBL_DIST_SCREEN": "3", "IBL_DIST_2SM": "0"}, "retrieval_vs_reference or topk"),   # ... on one SM
    ({"IBL_DIST_SCREEN": "3", "IBL_DIST_2SM": "0", "IBL_DIST_BN": "128", "IBL_GEMM_MC": "1"}, "retrieval_vs_reference or topk"),
]
# the distance-screening variants also run the whole exact-ranking suite
RANKING_ENVS = {"IBL_DIST_SCREEN", "IBL_DIST_2SM"}


@pytest.mark.gpu
@pytest.mark.parametrize("env,expr", VARIANTS, ids=[",".join(f"{k}={v}" for k, v in e.items()) for e, _ in VARIANTS])
def test_variant_matches_references(env, expr):
    child_env = dict(os.environ)
    child_env.update(env)
    files = [os.path.join(ROOT, "tests", "test_gpu_parity.py")]
    if RANKING_ENVS & set(env):
        files.append(os.path.join(ROOT, "tests", "test_gpu_ranking.py"))
        expr = f"({expr}) or test_gpu_ranking.py"
    r = subprocess.run([sys.executable, "-m", "pytest", *files, "-q", "-x", "-k", expr, "-p", "no:cacheprovider"],
                       cwd=ROOT, env=child_env, capture_output=True, text=True, timeout=600)
    tail = (r.stdout + r.stderr)[-2000:]
    assert r.returncode == 0, tail
    assert " passed" in r.stdout and "failed" not in r.stdout, tail


@pytest.mark.gpu
def test_umma_sw128_operand_accepts_unaligned_start_and_odd_group_stride():
    """Halo staging reads nine tap views out of one TMA-written tile: starts that are 128-byte but not 1024-byte
    aligned, 8-row groups 10 rows apart, descriptor base_offset = 0 (tensor-core MMA, here wgmma)."""
    from openibl_b200.engine import Engine, _ptr, _stream
    from openibl_b200._cabi import check
    eng = Engine.get(0)
    g = torch.Generator(device="cuda").manual_seed(5)
    rows = 200
    A = torch.randint(-8, 9, (rows, 64), device="cuda", generator=g).to(torch.bfloat16)
    B = torch.randint(-8, 9, (64, 64), device="cuda", generator=g).to(torch.bfloat16)
    D = torch.empty(128, 64, device="cuda")
    m = torch.arange(128, device="cuda")
    for group_rows, s0 in ((8, 0), (10, 0), (10, 1), (10, 11), (10, 22), (12, 3)):
        idx = s0 + (m // 8) * group_rows + (m % 8)
        want = A[idx].float() @ B.float().t()
        check(eng.lib.ibl_debug_umma_strided(eng.h, _ptr(A), rows, _ptr(B), s0, group_rows, 0, _ptr(D), _stream(0)), "probe")
        torch.cuda.synchronize()
        assert torch.equal(D, want), (group_rows, s0)

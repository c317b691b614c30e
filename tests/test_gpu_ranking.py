"""Every ranking path of ibl_l2dist_topk against an exact fp64 ranking.

Tensor cores only SCREEN candidates; exact fp32 arithmetic DECIDES the ranking (DESIGN §3).  Four paths implement
that promise (the path of the last call is read back through Engine.dist_path, so a change of the thresholds that
select them cannot quietly skip one):

    0  exact fp32 on the CUDA cores      gemm mode 0, d % 64 != 0, or n_valid == 0
    1  single-pass fp16 screening        m > 128, k <= 12
    2  bf16x3 screening, running top-16  m <= 128, k <= 12
    3  bf16x3 dense tiles + row select   k > 12

Every result is checked by `check_ranking` against fp64 distances, with a per-pair allowance for fp32 rounding
noise (see `noise` below) and no loose absolute tolerance.  The adversarial families at the end are databases whose
rounding errors are coherent across a row, so that a screening error bound that assumes independent element errors
is wrong by orders of magnitude; they must still rank exactly."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

PATH_NAMES = {0: "fp32", 1: "single-pass fp16", 2: "bf16x3 top-16", 3: "bf16x3 dense"}


@pytest.fixture(scope="module")
def eng():
    from openibl_b200.engine import Engine
    e = Engine.get(0)
    e.set_gemm_mode(1)
    yield e
    e.set_gemm_mode(1)


def expected_path(mode, m, d, k, n_valid):
    if mode == 0 or d % 64 != 0 or n_valid == 0:
        return 0
    if k <= 12 and m > 128:
        return 1
    return 2 if k <= 12 else 3


# ---- the checker ------------------------------------------------------------------------------------------------

def noise(qn, xn, d):
    """Allowance for fp32 rounding between an fp32 distance and the exact one, pair (i, j):
        eps_ij = 2^-22 (|q_i|^2 + |x_j|^2) + 2^-22 sqrt(D) |q_i| |x_j|
    The first term covers the roundings of |q|^2, |x|^2, their sum and the final fma (a few ulps of the norms), the
    second the fp32 dot product of D terms: a random-walk model of its rounding errors, 4 sigma for the serial
    summation of the CUDA-core path (the re-scoring kernels' lane-strided sums stay well inside it).  Coherent
    rounding (every partial sum rounding the same way) can exceed it; the adversarial databases below keep their
    structured part narrow enough that fp32 arithmetic still separates their rows."""
    return 2.0 ** -22 * (qn[:, None] ** 2 + xn[None, :] ** 2) + 2.0 ** -22 * math.sqrt(d) * qn[:, None] * xn[None, :]


def fp64_dist(q, x):
    """Exact (fp64, differences first: no cancellation) squared distances [m, n] on the device."""
    out = torch.empty(q.shape[0], x.shape[0], dtype=torch.float64, device=q.device)
    x64 = x.double()
    for i0 in range(0, q.shape[0], 64):
        out[i0:i0 + 64] = torch.cdist(q[i0:i0 + 64].double(), x64, compute_mode="donot_use_mm_for_euclid_dist") ** 2
    return out


def check_ranking(q, db, k, dk, ik, idx_base=0, n_valid=None, what=""):
    """Asserts that (dk, ik) is the exact top-k of q against db[:n_valid]:
    - indices distinct and in [idx_base, idx_base + n_valid); padding is (inf, -1), exactly where n_valid < k;
    - every distance within eps of the fp64 distance of its own index; distances ascending; equal fp32 distances
      in ascending index order;
    - no row left out whose fp64 distance is below the returned k-th by more than eps_row + eps_kth;
    - position by position, the fp64 ranking (ties to the lowest index) up to eps-ties."""
    m, d = q.shape
    nv = db.shape[0] if n_valid is None else n_valid
    assert dk.shape == (m, k) and ik.shape == (m, k), what
    v = min(k, nv)
    pad_i, pad_d = ik[:, v:], dk[:, v:]
    assert (pad_i == -1).all() and (torch.isinf(pad_d) & (pad_d > 0)).all(), f"{what}: padding is not (inf, -1)"
    if v == 0:
        return
    got = ik[:, :v] - idx_base
    assert ((got >= 0) & (got < nv)).all(), f"{what}: index out of range"
    srt = got.sort(dim=1).values
    assert (srt[:, 1:] != srt[:, :-1]).all(), f"{what}: repeated index"
    x = db[:nv]
    exact = fp64_dist(q, x)
    eps = noise(q.double().norm(dim=1), x.double().norm(dim=1), d)
    e_got, eps_got = exact.gather(1, got), eps.gather(1, got)
    gd = dk[:, :v].double()
    bad = (gd - e_got).abs() > eps_got
    if bad.any():
        i, j = [int(t) for t in bad.nonzero()[0]]
        raise AssertionError(f"{what}: query {i} rank {j} row {int(got[i, j])}: distance {float(gd[i, j]):.9g}, "
                             f"exact {float(e_got[i, j]):.9g}, allowance {float(eps_got[i, j]):.3g}")
    assert (gd[:, 1:] >= gd[:, :-1]).all(), f"{what}: distances not ascending"
    same = gd[:, 1:] == gd[:, :-1]
    assert (got[:, 1:][same] > got[:, :-1][same]).all(), f"{what}: equal distances not in index order"
    # completeness: nothing left out that is clearly nearer than the returned k-th
    left_out = torch.ones_like(exact, dtype=torch.bool).scatter_(1, got, False)
    missed = left_out & (exact < e_got[:, -1:] - (eps + eps_got[:, -1:]))
    if missed.any():
        i, j = [int(t) for t in missed.nonzero()[0]]
        raise AssertionError(f"{what}: query {i}: row {j} (exact {float(exact[i, j]):.6g}) left out, returned k-th "
                             f"row {int(got[i, -1])} has exact {float(e_got[i, -1]):.6g}")
    # the fp64 ranking, ties to the lowest index (stable sort), up to eps-ties
    want = torch.sort(exact, dim=1, stable=True).indices[:, :v]
    tie = (exact.gather(1, want) - e_got).abs() <= eps.gather(1, want) + eps_got
    wrong = (want != got) & ~tie
    if wrong.any():
        i, j = [int(t) for t in wrong.nonzero()[0]]
        raise AssertionError(f"{what}: query {i} rank {j}: row {int(got[i, j])} (exact {float(e_got[i, j]):.6g}), "
                             f"fp64 ranking has row {int(want[i, j])} (exact {float(exact[i, want[i, j]]):.6g})")


def rank(eng, q, db, k, mode=1, idx_base=0, n_valid=None, what=""):
    """One ibl_l2dist_topk call in gemm mode `mode`; asserts the path it took and the ranking."""
    nv = db.shape[0] if n_valid is None else n_valid
    eng.set_gemm_mode(mode)
    try:
        dk, ik = eng.l2dist_topk(q, db, k, idx_base=idx_base, n_valid=nv)
        path = eng.dist_path()
        flagged = eng.dist_flagged()
    finally:
        eng.set_gemm_mode(1)
    want = expected_path(mode, q.shape[0], q.shape[1], k, nv)
    tag = f"{what} [{PATH_NAMES.get(path, path)}, m={q.shape[0]} n={db.shape[0]} n_valid={nv} d={q.shape[1]} k={k}]"
    assert path == want, f"{tag}: expected the {PATH_NAMES[want]} path"
    # the guard's count describes this call: -1 on the exact path, 0..m on the screening paths
    assert (flagged == -1) if path == 0 else (0 <= flagged <= q.shape[0]), f"{tag}: dist_flagged() = {flagged}"
    check_ranking(q, db, k, dk, ik, idx_base, nv, tag)
    return dk, ik, path


def rank_all_paths(eng, q, db, k, idx_base=0, n_valid=None, what=""):
    """The case on every path that applies: the tensor-core path its shape selects, the same queries padded past
    or cut to the 128-query boundary (single pass vs bf16x3 top-16, k <= 12), and exact fp32.  Returns the set of
    paths taken."""
    seen = {rank(eng, q, db, k, 1, idx_base, n_valid, what)[2], rank(eng, q, db, k, 0, idx_base, n_valid, what)[2]}
    m = q.shape[0]
    if k <= 12 and q.shape[1] % 64 == 0:
        other = q[:128] if m > 128 else q.repeat(129 // m + 1, 1)[:max(129, m)]
        seen.add(rank(eng, other.contiguous(), db, k, 1, idx_base, n_valid, what + " (other side of m = 128)")[2])
    return seen


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def unit_rows(n, d, g):
    return torch.nn.functional.normalize(torch.randn(n, d, device="cuda", generator=g), dim=1)


def gallery(n, m, d, seed, sigma=0.3):
    """Queries near database rows (a retrieval-like set: clear nearest neighbours, crowded runners-up)."""
    g = gen(seed)
    db = unit_rows(n, d, g)
    q = db[torch.randint(0, n, (m,), device="cuda", generator=g)] + sigma * unit_rows(m, d, g)
    return q.contiguous(), db.contiguous()


# ---- edge catalogue ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [1, 16, 17, 127, 128, 129, 5000])
@pytest.mark.parametrize("m", [1, 9, 128, 129, 300])
def test_shapes(eng, m, n):
    """Query counts around the 128-row query tile, database sizes around the 16 candidates and the 128-row database
    tile (5000: several work items per query tile and the shared gate), every k class."""
    q, db = gallery(n, m, 64, seed=m * 7919 + n)
    for k in (1, 10, 12, 13, 128):
        rank_all_paths(eng, q, db, k, what="shapes")


@pytest.mark.parametrize("d", [64, 100, 512, 4096, 32768])
def test_dims(eng, d):
    """100: d % 64 != 0 (exact fp32 route); 32768: the raw-VLAD width, query rows not staged in shared memory."""
    for m, n in ((9, 1000), (200, 1000), (150, 129)):
        q, db = gallery(n, m, d, seed=d + m)
        for k in (1, 12, 13):
            paths = rank_all_paths(eng, q, db, k, what="dims")
            tc = {1, 2} if k <= 12 else {3}
            assert paths == ({0} if d % 64 else {0} | tc), paths


@pytest.mark.parametrize("idx_base", [0, 5000, 2 ** 31 + 7])
@pytest.mark.parametrize("m", [9, 300])
def test_ragged_shards(eng, m, idx_base):
    """n_valid < n (wrap-around padding), n_valid <= 16, n_valid < k (padded with (inf, -1)), n_valid = 0."""
    q, db = gallery(700, m, 256, seed=m + 11)
    db[600:] = q[: 100 if m > 100 else m].repeat(100, 1)[:100]      # padding rows nearer than anything: ignored
    for nv in (700, 600, 333, 17, 16, 5, 1, 0):
        for k in (1, 10, 12, 13):
            rank_all_paths(eng, q, db, k, idx_base, nv, what="ragged")


def mixed_rows(n, d, g):
    """Unit rows scaled by powers of two (2^-10 .. 2^10) and by non-powers of two."""
    scales = torch.tensor([2.0 ** -10, 0.37, 1.0, 3.3, 2.0 ** 10, 1e-3, 77.7], device="cuda")
    s = scales[torch.randint(0, len(scales), (n, 1), device="cuda", generator=g)]
    return (unit_rows(n, d, g) * s).contiguous()


@pytest.mark.parametrize("d", [512, 4096])
def test_magnitudes(eng, d):
    """Whole sets scaled by 2^+-10 and by non-powers of two; mixed-magnitude rows; a zero query and a zero database
    row; rows with one huge element (the rest of the row falls into the fp16 subnormals after scaling); duplicates."""
    g = gen(d)
    q0, db0 = gallery(3000, 200, d, seed=d + 1)
    for s in (2.0 ** 10, 2.0 ** -10, 0.3, 37.5):
        rank_all_paths(eng, (q0 * s).contiguous(), (db0 * s).contiguous(), 10, what=f"scaled {s}")
    db = mixed_rows(3000, d, g)
    q = torch.cat([db[:150] * (1 + 1e-3 * torch.randn(150, 1, device="cuda", generator=g)), mixed_rows(50, d, g)])
    q[7] = 0
    db[100] = 0
    spike = db[200:210].clone() * 1e-3
    spike[:, 5] = 1e3
    db[200:210] = spike
    q[20:25] = spike[:5] * (1 + 2 ** -12)
    db[2990:] = db[:10]                                              # exact duplicates: ties to the lower index
    q = q.contiguous()
    for k in (1, 10, 13):
        rank_all_paths(eng, q, db, k, what="mixed magnitudes")


def test_duplicates_keep_index_order(eng):
    """Identical rows give identical fp32 distances on every path: the lower index must come first."""
    q, db = gallery(50, 160, 512, seed=4)
    dup = torch.cat([db, db, db]).contiguous()
    for k in (3, 12, 13):
        for mode in (1, 0):
            for qq in (q, q[:100].contiguous()):
                _, ik, _ = rank(eng, qq, dup, k, mode, what="duplicates")
                assert (ik[:, 1] == ik[:, 0] + 50).all() and (ik[:, 2] == ik[:, 0] + 100).all()


@pytest.mark.parametrize("k", [10, 13])
def test_many_exact_ties_overflow_the_fallback_list(eng, k):
    """400 identical rows nearest to every query: the guard must list every query (16 or k + 8 survivors cannot
    settle 400 ties), and more rows lie within the k-th distance than the exact fallback's per-query list holds, so
    its blockwise scan ranks them: lowest indices first."""
    q, db = gallery(3000, 1, 512, seed=9)
    db[1000:1400] = q[0] + 0.01 * unit_rows(1, 512, gen(10))
    for m in (64, 160):
        qq = q.repeat(m, 1).contiguous()
        for mode in (1, 0):
            _, ik, path = rank(eng, qq, db, k, mode, what="400 ties")
            assert (ik == torch.arange(1000, 1000 + k, device="cuda")).all(), PATH_NAMES[path]
            assert eng.dist_flagged() == (m if path else -1), PATH_NAMES[path]


def test_workspace_reuse_across_shapes(eng):
    """Back-to-back calls on one engine, shapes decreasing then increasing: the workspaces, the shared-gate memset
    and the guard's counter are reused without stale state leaking into the next call."""
    shapes = [(300, 5000, 4096), (200, 1000, 512), (129, 17, 64), (129, 200, 1024), (400, 8000, 2048)]
    for i, (m, n, d) in enumerate(shapes + shapes[::-1]):
        q, db = gallery(n, m, d, seed=100 + i)
        for k in (1, 12):
            assert rank(eng, q, db, k, what="reuse")[2] == expected_path(1, m, d, k, n)
        rank(eng, q[:64].contiguous(), db, 10, what="reuse")


@pytest.mark.parametrize("k", [10, 13])
@pytest.mark.parametrize("m", [9, 300])
def test_shard_merge_equals_whole(eng, m, k):
    """Per-shard top-k (idx_base = shard offset, ragged last shard) merged with topk_merge == whole-database top-k."""
    q, db = gallery(5000, m, 512, seed=m + k)
    bounds = [0, 1300, 2600, 3900, 5000]
    parts = []
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        shard = torch.zeros(1300, 512, device="cuda")
        shard[:hi - lo] = db[lo:hi]
        parts.append(eng.l2dist_topk(q, shard, k, idx_base=lo, n_valid=hi - lo))
    md, mi = eng.topk_merge(torch.stack([p[0] for p in parts]), torch.stack([p[1] for p in parts]), k)
    check_ranking(q, db, k, md, mi, what="merged shards")
    wd, wi, _ = rank(eng, q, db, k, what="whole")
    assert torch.equal(mi, wi) and torch.equal(md, wd)


# ---- adversarial families: coherent rounding errors ---------------------------------------------------------------

def coherent_block(rows, d, value, p):
    """rows x d, `value` in the first p columns, zero elsewhere."""
    x = torch.zeros(rows, d, device="cuda")
    x[:, :p] = value
    return x


def fp16_family(d, k, g):
    """q = 2^-7 on P = min(d, 4096) elements.  The true nearest row X = 2^-7 (1 + 2^-11) there sits exactly halfway
    between two fp16 values after per-row power-of-two scaling and rounds down onto q: exact distance P 2^-36,
    screened P 2^-24 (every element's rounding error has the same sign).  Decoys lower c < P/16 elements by 2^-10;
    they are exact in fp16, at exact distances c 2^-20 -- below X's screened distance, far above its exact one.
    k + 24 decoys push X out of any candidate list that is k + 8 or 16 long.  Far rows fill the rest."""
    p = min(d, 4096)
    q = coherent_block(1, d, 2.0 ** -7, p)
    x = coherent_block(1, d, 2.0 ** -7 * (1 + 2.0 ** -11), p)
    decoys = q.repeat(k + 24, 1)
    for j in range(k + 24):
        c = 1 + (j * 5) % (p // 32)
        cols = (torch.arange(c, device="cuda") + 13 * j) % p
        decoys[j, cols] -= 2.0 ** -10
    return q, x, decoys


def bf16_family(d, k, g):
    """q = X = 2^-7 (1 + 2^-8) on P = 128 elements: hi = 2^-7, lo = 2^-15, so the dropped lo.lo term puts X's
    screened distance at 2 P 2^-30 against an exact 0.  Decoys have bf16-exact (lo = 0) elements 2^-7 or
    2^-7 - 2^-14 (c < P/8 of them), exact and screened distance (P + 8c) 2^-30 < 2 P 2^-30.  With P = 128 every fp32
    sum over these rows is exact, so each path's fp32 arithmetic puts X (0) first: a miss is a wrong answer, not a
    near-tie."""
    p = 128
    q = coherent_block(1, d, 2.0 ** -7 * (1 + 2.0 ** -8), p)
    x = q.clone()
    decoys = coherent_block(k + 24, d, 2.0 ** -7, p)
    for j in range(k + 24):
        c = j % (p // 8)
        cols = (torch.arange(c, device="cuda") + 29 * j) % p
        decoys[j, cols] -= 2.0 ** -14
    return q, x, decoys


def adversarial_db(family, d, k, hidden, seed):
    g = gen(seed)
    q, x, decoys = (fp16_family if family == "fp16" else bf16_family)(d, k, g)
    coherent = torch.cat([decoys[: len(decoys) // 2], x, decoys[len(decoys) // 2:]])
    if hidden:                              # hidden among 10k random unit rows
        filler = unit_rows(10000, d, g)
    else:                                   # among rows near q that are clearly farther than every decoy
        filler = q + 0.01 * torch.randn(200, d, device="cuda", generator=g)
    n = len(filler) + len(coherent)
    pos = torch.randperm(n, device="cuda", generator=g)[: len(coherent)].sort().values
    db = torch.empty(n, d, device="cuda")
    keep = torch.ones(n, dtype=torch.bool, device="cuda")
    keep[pos] = False
    db[pos] = coherent
    db[keep] = filler
    return q, db.contiguous(), int(pos[len(decoys) // 2])


@pytest.mark.parametrize("k", [1, 10, 120])
@pytest.mark.parametrize("d", [512, 4096, 32768])
@pytest.mark.parametrize("family,hidden", [("fp16", False), ("bf16x3", False), ("fp16", True), ("bf16x3", True)],
                         ids=["fp16", "bf16x3", "fp16-hidden", "bf16x3-hidden"])
def test_coherent_rounding_ranks_exactly(eng, family, hidden, d, k):
    """The true nearest row must come first on every path, with the queries repeated so that m lands on both sides
    of 128 (bf16x3 top-16 and single pass for k <= 12; bf16x3 dense for k = 120)."""
    q1, db, ix = adversarial_db(family, d, k, hidden, seed=d + k)
    for m in (64, 192):
        q = q1.repeat(m, 1).contiguous()
        for mode in (1, 0):
            dk, ik, path = rank(eng, q, db, k, mode, what=f"{family}{' hidden' if hidden else ''}")
            assert (ik[:, 0] == ix).all(), f"{PATH_NAMES[path]}: the true nearest row {ix} is not first"

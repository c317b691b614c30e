"""CPU model of the tensor-core screening arithmetic of ibl_l2dist_topk and of the guard that decides whether the
screened candidate list can be trusted (runs without a GPU).

The kernels keep, per query, the candidates with the smallest SCREENED distances, re-score them in exact fp32 and
rank those.  A row that was not kept has a screened distance >= s (the last kept screened distance); if its exact
distance is >= s - B, and s - B > e_k (the k-th exact distance), it cannot belong in the top-k.  So B must bound the
screening error |screened - exact| for every pair; otherwise the guard does not fire and the answer is wrong.

Here the operands are rounded exactly as the kernels round them and the products are summed in fp64, so the
emulated error is the OPERAND rounding error.  The guard formulas below mirror the kernels' constants; the operand
part of each must bound the emulated error on any data, including databases whose rounding errors are coherent
across a row (all of one sign), where a bound that assumes independent element errors fails."""
import math

import pytest
import torch

from openibl_b200 import synth

U23 = 2.0 ** -23
ACC_KAPPA = 8.0          # D1_ACC_KAPPA


# ---- operand rounding, as the kernels do it ---------------------------------------------------------------------

def fp16_planes(x):
    """rows_f16_kernel (tc_dist1.cu): per-row scale 2^e with the row max in [0.5, 1) (frexp), plane = fp16 RN of
    x * 2^-e (subnormals included).  Returns (operand as seen by the MMA, in fp64, residual norm |x - operand|)."""
    x = x.float()
    mx = x.abs().amax(dim=1)
    e = torch.where((mx > 0) & torch.isfinite(mx), torch.frexp(mx).exponent, torch.zeros_like(mx, dtype=torch.int32))
    sc = torch.ldexp(torch.ones_like(mx, dtype=torch.float64), e.double())
    op = (x * torch.ldexp(torch.ones_like(mx), -e.float())[:, None]).half().double() * sc[:, None]
    return op, (x.double() - op).norm(dim=1)


def bf16_split(x):
    """planes_sqnorm_kernel (gemm_simt.cu): hi = bf16 RN(x), lo = bf16 RN(x - hi).  Returns (hi, lo, |lo|,
    |x - hi - lo|) in fp64."""
    x = x.float()
    hi = x.bfloat16().float()
    lo = (x - hi).bfloat16().float()
    r = x.double() - hi.double() - lo.double()
    return hi.double(), lo.double(), lo.double().norm(dim=1), r.norm(dim=1)


def screened_fp16(q, db):
    """Distance screened by gemm_f16_top16_kernel, operand rounding only: |q|^2 + |d|^2 - 2 q~.d~."""
    qo, _ = fp16_planes(q)
    do, _ = fp16_planes(db)
    return sqn(q)[:, None] + sqn(db)[None] - 2 * qo @ do.t()


def screened_bf16x3(q, db):
    """Distance screened by gemm_tc_kernel (tc_gemm.cu): lo.hi + hi.lo + hi.hi, the lo.lo term dropped."""
    qh, ql, _, _ = bf16_split(q)
    dh, dl, _, _ = bf16_split(db)
    return sqn(q)[:, None] + sqn(db)[None] - 2 * (qh @ dh.t() + qh @ dl.t() + ql @ dh.t())


def sqn(x):
    return (x.double() ** 2).sum(1)


def exact(q, db):
    q, db = q.double(), db.double()
    return sqn(q)[:, None] + sqn(db)[None] - 2 * q @ db.t()


# ---- the guard formulas -----------------------------------------------------------------------------------------

def guard_bound(q_sq, q_lo, q_res, db_sq_max, db_lo_max, db_res_max, d, mmas_per_k16, operand_only=False):
    """d1_screen_bound (tc_dist1.cu), used by dist_finish_kernel (single pass: no lo plane, one MMA per 16-wide
    K step) and dist_guard_kernel (bf16x3: three MMAs per K step).  With x = op(x) + r (op = what the MMA sees:
    scaled fp16, or hi + lo) and the dropped lo.lo term,
        |q.d - screened dot| <= |lo_q| |lo_d| + |q| |r_d| + |r_q| |d| + |r_q| |r_d|     (Cauchy-Schwarz, rigorous)
    per pair, with the database side replaced by its maximum over the rows.  Statistical, not a bound: the fp32
    accumulation inside the tensor core, 8 sigma of a random walk of one 2^-24 rounding per accumulator update (one
    per MMA and 16-wide K step) relative to (|q| + |lo_q| + |r_q|)(max|d| + max|lo_d| + max|r_d|).  Then the
    epilogue's fma (2^-23 (|q|^2 + max|d|^2)), distance = -2 dot, and (1 + d 2^-23) for the fp32 evaluation of the
    bound."""
    nq, dm = math.sqrt(q_sq), math.sqrt(db_sq_max)
    dot = q_lo * db_lo_max + nq * db_res_max + q_res * dm + q_res * db_res_max
    if operand_only:
        return 2 * dot
    acc = ACC_KAPPA * 2.0 ** -24 * math.sqrt(d / 16 * mmas_per_k16) * (nq + q_lo + q_res) * (dm + db_lo_max + db_res_max)
    return (2 * (dot + acc) + U23 * (q_sq + db_sq_max)) * (1 + d * U23)


def fp16_bounds(q, db, operand_only=False):
    _, rq = fp16_planes(q)
    _, rd = fp16_planes(db)
    dsq = float(sqn(db).max())
    return torch.tensor([guard_bound(float(a), 0.0, float(r), dsq, 0.0, float(rd.max()), q.shape[1], 1, operand_only)
                         for a, r in zip(sqn(q), rq)], dtype=torch.float64)


def bf16_bounds(q, db, operand_only=False):
    _, _, lq, rq = bf16_split(q)
    _, _, ld, rd = bf16_split(db)
    dsq = float(sqn(db).max())
    return torch.tensor([guard_bound(float(a), float(l), float(r), dsq, float(ld.max()), float(rd.max()), q.shape[1], 3,
                                     operand_only) for a, l, r in zip(sqn(q), lq, rq)], dtype=torch.float64)


def old_fp16_guard(q, db):
    """The single-pass guard before it bounded anything: 8 sigma of independent fp16 rounding errors from the
    rows' 4-norms, plus a subnormal term.  Kept to show that the coherent family below defeats it."""
    c = 8.0 * 2.0 * 1.41421356 * 0.41 * 4.8828125e-4
    q4, d4 = (q.double() ** 4).sum(1) ** 0.25, (db.double() ** 4).sum(1) ** 0.25
    qmax, dmax = q.double().abs().amax(1), db.double().abs().amax(1)
    return c * q4 * d4.max() + 2 * 5.9604645e-8 * math.sqrt(q.shape[1]) * (dmax.max() * sqn(q).sqrt() +
                                                                          qmax * sqn(db).max().sqrt())


# ---- data -------------------------------------------------------------------------------------------------------

def fp16_family(d, k=10):
    """As in test_gpu_ranking.py: q = 2^-7, X = 2^-7 (1 + 2^-11) rounds onto q in fp16, decoys exact in fp16."""
    q = torch.full((1, d), 2.0 ** -7)
    x = torch.full((1, d), 2.0 ** -7 * (1 + 2.0 ** -11))
    dec = q.repeat(k + 24, 1)
    for j in range(k + 24):
        c = 1 + (j * 5) % max(2, d // 32)
        dec[j, (torch.arange(c) + 13 * j) % d] -= 2.0 ** -10
    return q, torch.cat([x, dec])


def bf16_family(d, k=10):
    """q = X = 2^-7 (1 + 2^-8): lo.lo dropped; decoys bf16-exact."""
    q = torch.full((1, d), 2.0 ** -7 * (1 + 2.0 ** -8))
    dec = torch.full((k + 24, d), 2.0 ** -7)
    for j in range(k + 24):
        c = (j * 16) % max(2, d // 16)
        dec[j, (torch.arange(c) + 29 * j) % d] -= 2.0 ** -14
    return q, torch.cat([q.clone(), dec])


def data(kind, n, d, g):
    if kind == "random":
        return torch.randn(n, d, generator=g)
    if kind == "quantised":                          # uint8-like codes
        return torch.randint(0, 256, (n, d), generator=g).float()
    if kind == "sparse":
        x = torch.randn(n, d, generator=g)
        return x * (torch.rand(n, d, generator=g) < 0.05)
    if kind == "same-sign":
        return torch.randn(n, d, generator=g).abs() * 1e-3
    if kind == "spike":                              # one huge element: the rest falls into the fp16 subnormals
        x = torch.randn(n, d, generator=g) * 1e-4
        x[:, 3] = 1e4
        return x
    raise ValueError(kind)


FAMILIES = {"fp16-coherent": fp16_family, "bf16x3-coherent": bf16_family}


@pytest.mark.parametrize("d", [512, 4096, 32768])
@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_guard_bounds_coherent_rounding(family, d):
    q, db = FAMILIES[family](d)
    for screened, bounds in ((screened_fp16, fp16_bounds), (screened_bf16x3, bf16_bounds)):
        err = (screened(q, db) - exact(q, db)).abs().amax(dim=1)
        assert (bounds(q, db, operand_only=True) >= err).all(), (screened.__name__, err)
    if family == "fp16-coherent":
        # the nearest row X is screened d 2^-24 away from its exact distance, far beyond the old statistical bound
        err = (screened_fp16(q, db) - exact(q, db)).abs()[0, 0]
        assert abs(float(err) - d * 2.0 ** -24) < 1e-3 * d * 2.0 ** -24
        assert float(old_fp16_guard(q, db)[0]) < 0.5 * float(err)
    else:
        err = (screened_bf16x3(q, db) - exact(q, db)).abs()[0, 0]
        assert abs(float(err) - 2 * d * 2.0 ** -30) < 1e-3 * d * 2.0 ** -30


@pytest.mark.parametrize("kind", ["random", "quantised", "sparse", "same-sign", "spike"])
@pytest.mark.parametrize("d", [64, 4096])
def test_guard_bounds_random_data(kind, d):
    g = torch.Generator().manual_seed(d + len(kind))
    q, db = data(kind, 24, d, g), data(kind, 200, d, g)
    q[:4] = db[:4] * (1 + 2.0 ** -12)                   # near-duplicates: the smallest distances
    for screened, bounds in ((screened_fp16, fp16_bounds), (screened_bf16x3, bf16_bounds)):
        err = (screened(q, db) - exact(q, db)).abs().amax(dim=1)
        b = bounds(q, db, operand_only=True)
        assert (b >= err).all(), (kind, screened.__name__, float((err / b).max()))
        # and not vacuous: within a few hundred of the worst observed error on unstructured data
        if kind == "random":
            assert (b <= 400 * err).all(), (kind, screened.__name__, float((b / err).max()))


def flag_rate(q, db, k, screened, bounds, keep):
    """Emulated guard decision per query: s = the keep-th smallest screened distance, e_k = the k-th exact distance
    among the kept rows; the query falls back to exact brute force when s - B <= e_k."""
    scr = screened(q, db)
    ex = exact(q, db)
    s = scr.sort(dim=1)
    kept = s.indices[:, :keep]
    e_k = ex.gather(1, kept).sort(dim=1).values[:, k - 1]
    return int((s.values[:, keep - 1] - bounds(q, db) <= e_k).sum())


@pytest.mark.parametrize("d,n_db,n_q", [(512, 10000, 300), (4096, 10000, 300), (32768, 2000, 200)])
def test_guard_firing_rate_on_descriptor_like_data(d, n_db, n_q):
    """Retrieval-like data (synth.make_gallery, sigma 0.25): the rigorous bound must leave the fast path alone at
    the benchmark's width (4096) and fall back for a small share of queries at the raw-VLAD width."""
    torch.set_num_threads(max(1, torch.get_num_threads()))
    q, db, _ = synth.make_gallery(n_db, n_q, d)
    single = flag_rate(q, db, 10, screened_fp16, fp16_bounds, 16)
    top16 = flag_rate(q, db, 10, screened_bf16x3, bf16_bounds, 16)
    dense = flag_rate(q, db, 120, screened_bf16x3, bf16_bounds, 128)
    print(f"\nd={d}: guard fires (emulated) single-pass {single}/{n_q}, bf16x3 top-16 {top16}/{n_q}, "
          f"bf16x3 dense k=120 {dense}/{n_q}")
    if d <= 4096:
        assert single == 0 and top16 == 0 and dense == 0
    else:
        assert single <= n_q // 4 and top16 <= n_q // 4

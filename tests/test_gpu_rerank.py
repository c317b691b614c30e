"""k-reciprocal re-ranking on sparse data (ibl_knn_rowmax + ibl_rerank_topk, evaluators.sharded_rerank_topk) against
the reference function (tests/golden/rerank.npz) and against the dense re_ranking of openibl_b200/utils/rerank.py."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from openibl_b200.engine import Engine
    return Engine.get(0)


def _half(k1):
    return int(np.around(k1 / 2.0))


def _sparse(eng, q, db, k1, k2, lam, k):
    """world size 1 through the public host function"""
    from openibl_b200.evaluators import sharded_rerank_topk
    q, db = q.cuda().float().contiguous(), db.cuda().float().contiguous()
    fd, fi = sharded_rerank_topk(q, db, k, 0, db.shape[0], k1=k1, k2=k2, lambda_value=lam)
    return fd.cpu(), fi.cpu()


def _d64(a, b):
    a, b = a.double(), b.double()
    return (a * a).sum(1, keepdim=True) + (b * b).sum(1)[None] - 2 * a @ b.t()


def _dense_ref(eng, q, db, k1, k2, lam, k, want_final=False):
    """dense re_ranking fed fp64-accurate distances, ranked by ibl_topk_rows"""
    from openibl_b200.utils.rerank import re_ranking
    q, db = q.float(), db.float()
    qg, qq, gg = _d64(q, db).float(), _d64(q, q).float(), _d64(db, db).float()
    final = re_ranking(qg.cuda(), qq.cuda(), gg.cuda(), k1=k1, k2=k2, lambda_value=lam)
    fd, fi = eng.topk_rows(final.contiguous(), min(k, db.shape[0]))
    if want_final:
        return fd.cpu(), fi.cpu(), final.cpu()
    return fd.cpu(), fi.cpu()


def _margins_ok(q, db, k1, gap=1e-4):
    """every row's neighbour-list boundaries (ranks k1+1 / k1+2 and the half width) separated by more than gap"""
    X = torch.cat([q, db]).double()
    d2 = _d64(X, X) ** 2
    d2 = d2 / d2.max(dim=1, keepdim=True).values
    s = torch.sort(d2, dim=1).values
    cuts = [k1 + 1, _half(k1) + 1]
    return all(bool(((s[:, c] - s[:, c - 1]) > gap).all()) for c in cuts if c < s.shape[1])


def _clustered(n_q, n_db, d, seed, clusters=None):
    g = torch.Generator().manual_seed(seed)
    clusters = clusters or max(2, (n_q + n_db) // 12)
    cent = torch.randn(clusters, d, generator=g)
    X = cent[torch.randint(0, clusters, (n_q + n_db,), generator=g)] + 0.35 * torch.randn(n_q + n_db, d, generator=g)
    X = X / X.norm(dim=1, keepdim=True)
    return X[:n_q].contiguous(), X[n_q:].contiguous()


def test_reference_golden(eng):
    """d = 16 / 24 (the d % 64 != 0 path) against the unmodified reference function's final matrix"""
    g = load_golden("rerank")
    for name in "abc":
        k1, k2, lam = g[f"{name}_params"]
        q, db = torch.from_numpy(g[f"{name}_q"]), torch.from_numpy(g[f"{name}_db"])
        ref = torch.from_numpy(g[f"{name}_final"])
        k = min(128, db.shape[0])
        fd, fi = _sparse(eng, q, db, int(k1), int(k2), float(lam), k)
        want = torch.sort(ref, dim=1, stable=True)
        close = ((fd - want.values[:, :k]).abs() < 1e-4).float().mean()
        assert close > 0.995, (name, float(close))
        got_vals = torch.gather(ref, 1, fi)               # the reference's value at each returned row
        assert float(((got_vals - fd).abs() < 1e-4).float().mean()) > 0.995, name
        assert float((fi[:, 0] == want.indices[:, 0]).float().mean()) > 0.95, name


def _separated(n_clusters, n_q, d, k1, seed):
    """Data whose neighbour lists have margins: clusters of k1 + 1 rows, each on its own pair of coordinate axes
    (centre +-1.5 on the first, positions on the second).  A cluster is a tight group of round(k1/2) + 1 rows at
    0 .. 0.2 and a second group at 1.0 .. 1.2, so every row's first k1 + 1 neighbours are its cluster and its first
    round(k1/2) + 1 are its group, or its group and the nearest row of the other one; the positions are stretched
    unevenly so that no two distances in a cluster tie.  Rows are shuffled before the query / gallery split."""
    s, h = k1 + 1, _half(k1)
    assert n_clusters <= d
    pos = torch.cat([torch.arange(h + 1) * 0.02, 1.0 + torch.arange(k1 - h) * 0.02]).double()
    pos = pos * (1 + 0.01 * torch.arange(s).double())
    X = torch.zeros(n_clusters, s, d, dtype=torch.float64)
    for c in range(n_clusters):
        X[c, :, (c // 2) * 2] = 1.5 if c % 2 == 0 else -1.5
        X[c, :, (c // 2) * 2 + 1] = pos
    X = X.reshape(-1, d)
    X = X[torch.randperm(X.shape[0], generator=torch.Generator().manual_seed(seed))].float()
    return X[:n_q].contiguous(), X[n_q:].contiguous()


@pytest.mark.parametrize("d,n_clusters,n_q,k1,k2,lam", [
    (64, 10, 9, 2, 1, 0.3),
    (64, 30, 33, 10, 6, 0.0),
    (64, 28, 63, 20, 1, 0.1),
    (64, 18, 52, 25, 6, 1.0),
    (4096, 96, 216, 20, 6, 0.3),
    (4096, 454, 506, 10, 1, 0.0),
    (64, 11, 21, 20, 21, 0.3),            # k2 = k1 + 1
])
def test_agrees_with_dense_path(eng, d, n_clusters, n_q, k1, k2, lam):
    """Exact agreement where the fp64 neighbour lists have margins: values within 2e-6, identical top-k indices.

    With k2 > 1, rows that share their first k2 neighbours have mathematically identical V rows, and so queries see
    exact ties in the final distance; which of the tied rows comes first is decided by the last bit of two
    differently ordered fp32 sums (the unmodified reference and the dense torch path order such ties differently
    from each other too).  There the indices must be a ranking of the dense final matrix up to ties of 3e-7."""
    q, db = _separated(n_clusters, n_q, d, k1, seed=n_clusters + k1)
    assert _margins_ok(q, db, k1)
    k = min(10, db.shape[0])
    fd, fi = _sparse(eng, q, db, k1, k2, lam, k)
    rd, ri, final = _dense_ref(eng, q, db, k1, k2, lam, k, want_final=True)
    assert float((fd - rd).abs().max()) < 2e-6
    if k2 == 1:
        assert torch.equal(fi, ri), float((fi == ri).float().mean())
    else:
        assert float((torch.gather(final, 1, fi) - rd).abs().max()) <= 3e-7      # each returned row is rank-correct


def test_clustered_data_without_margins(eng):
    """Overlapping clusters: near-ties in the neighbour lists; the bulk of the ranking agrees with the dense path."""
    q, db = _clustered(60, 500, 64, seed=5)
    fd, fi = _sparse(eng, q, db, 20, 6, 0.3, 10)
    rd, ri = _dense_ref(eng, q, db, 20, 6, 0.3, 10)
    assert float((fi == ri).float().mean()) >= 0.99


def test_random_data_recalls(eng):
    from openibl_b200 import synth
    q, db, gt = synth.make_gallery(n_db=1500, n_q=150, dim=256, sigma=0.6)
    fd, fi = _sparse(eng, q, db, 20, 6, 0.3, 10)
    rd, ri = _dense_ref(eng, q, db, 20, 6, 0.3, 10)
    assert float((fi == ri).float().mean()) >= 0.99
    for n in (1, 5, 10):
        a = (fi[:, :n] == gt[:, None]).any(1).float().mean()
        b = (ri[:, :n] == gt[:, None]).any(1).float().mean()
        assert float(a) == float(b), n


def test_edge_cases(eng):
    q, db = _clustered(20, 120, 64, seed=7)
    # duplicated rows: computed self/duplicate distances can be negative; lists sort by d^2
    db2 = torch.cat([db, db[:10], q[:3]])
    fd, fi = _sparse(eng, q, db2, 10, 1, 0.3, 10)
    rd, ri = _dense_ref(eng, q, db2, 10, 1, 0.3, 10)
    assert float((fi == ri).float().mean()) >= 0.97
    # many exact ties: quantised rows repeat
    qt = torch.round(q * 2) / 2
    dbt = torch.round(db * 2) / 2
    fd, fi = _sparse(eng, qt, dbt, 10, 6, 0.0, 10)
    rd, ri = _dense_ref(eng, qt, dbt, 10, 6, 0.0, 10)
    assert float((fd - rd).abs().max()) < 1e-5
    # lambda = 0: a query far from every gallery row has an empty overlap; its ranking is rows 0, 1, 2, ... (jac = 1)
    far = torch.zeros(1, 64)
    far[0, 0] = 50.0
    qe = torch.cat([q, far])
    fd, fi = _sparse(eng, qe, db, 10, 1, 0.0, 10)
    rd, ri = _dense_ref(eng, qe, db, 10, 1, 0.0, 10)
    assert torch.equal(fi[-1], torch.arange(10)) and bool((fd[-1] == 1.0).all())
    assert float((fi == ri).float().mean()) >= 0.97
    # m = 1, k = 120, N = k1 + 1
    fd, fi = _sparse(eng, q[:1], db, 10, 1, 0.3, 120)
    rd, ri = _dense_ref(eng, q[:1], db, 10, 1, 0.3, 120)
    assert float((fi == ri).float().mean()) >= 0.97 and fi.shape == (1, 120)
    fd, fi = _sparse(eng, q[:2], db[:9], 10, 1, 0.3, 5)
    rd, ri = _dense_ref(eng, q[:2], db[:9], 10, 1, 0.3, 5)
    assert torch.equal(fi, ri)
    with pytest.raises(ValueError):
        _sparse(eng, q[:2], db[:8], 10, 1, 0.3, 5)       # N < k1 + 1
    with pytest.raises(ValueError):
        _sparse(eng, q, db, 128, 1, 0.3, 5)              # k1 + 1 > 128
    from openibl_b200._cabi import IblError
    X = torch.cat([q, db]).cuda()
    with pytest.raises(IblError):
        eng.knn_rowmax(X, 129)


@pytest.mark.parametrize("d,N,adversarial", [(64, 700, False), (4096, 3000, False), (256, 1500, True)])
def test_rowmax_and_lists_vs_fp64(eng, d, N, adversarial):
    g = torch.Generator().manual_seed(N)
    X = torch.randn(N, d, generator=g)
    X = X / X.norm(dim=1, keepdim=True)
    if adversarial:                       # same-sign rows: every rounding error of a row points the same way
        X = X.abs() + 1.0
        X = X / X.norm(dim=1, keepdim=True)
    w = 21
    idx, dd, mx = eng.knn_rowmax(X.cuda(), w)
    idx, dd, mx = idx.cpu(), dd.cpu(), mx.cpu()
    D = _d64(X, X)
    M = (D * D).max(dim=1).values
    # the fp32 distance |x|^2 + |y|^2 - 2 x.y carries a few ulps of |x|^2 + |y|^2 (cancellation): allow 4 of them in d
    nrm = (X.double() ** 2).sum(1)
    delta = 4 * 2.0 ** -23 * (nrm + nrm.max())
    assert bool(((mx.double() - M).abs() <= 2 * M.sqrt() * delta + delta ** 2).all())
    s2, order = torch.sort(D * D, dim=1, stable=True)
    dsorted = D.gather(1, order)
    gap_ok = torch.ones(N, dtype=torch.bool)
    for c in range(1, w + 1):             # rows where every consecutive gap of the first w + 1 exceeds 2 delta in d
        gap_ok &= (dsorted[:, c].abs() - dsorted[:, c - 1].abs()) > 2 * delta
    if not adversarial:
        assert int(gap_ok.sum()) > N // 10
        assert torch.equal(idx[gap_ok], order[gap_ok, :w])
    # same-sign rows: the cancellation in |x|^2 + |y|^2 - 2 x.y leaves almost no gap above the fp32 noise, so only the
    # row maximum (above) and the listed distances (below) are checked there
    assert float((dd.double() - D.gather(1, idx)).abs().max()) < 1e-4


def test_multi_chunk_neighbour_pass_vs_fp64(eng):
    """N > 32768 columns: per-chunk near and far lists merged across chunks.  Odd row slices (the merged int64
    candidate array then starts at an odd multiple of 4 bytes) against fp64, and the same rows computed in a
    different slice bit-identical."""
    N, d, w = 100003, 64, 21
    g = torch.Generator().manual_seed(11)
    X = torch.randn(N, d, generator=g)
    X = (X / X.norm(dim=1, keepdim=True)).cuda()
    nrm = (X.double() ** 2).sum(1)
    for row0, n_rows in ((0, 5), (40000, 333), (N - 1027, 1027)):
        idx, dd, mx = eng.knn_rowmax(X, w, row0, n_rows)
        assert eng.knn_flagged() >= 0
        D = (X[row0:row0 + n_rows].double() @ X.double().t()).mul_(-2).add_(nrm[row0:row0 + n_rows, None]).add_(nrm)
        M = (D * D).max(dim=1).values
        delta = 4 * 2.0 ** -23 * (nrm[row0:row0 + n_rows] + nrm.max())
        assert bool(((mx.double() - M).abs() <= 2 * M.sqrt() * delta + delta ** 2).all())
        s2, order = torch.sort(D * D, dim=1, stable=True)
        dsorted = D.gather(1, order[:, :w + 1])
        gap_ok = torch.ones(n_rows, dtype=torch.bool, device=X.device)
        for c in range(1, w + 1):
            gap_ok &= (dsorted[:, c].abs() - dsorted[:, c - 1].abs()) > 2 * delta
        assert int(gap_ok.sum()) >= max(1, n_rows // 2)
        assert torch.equal(idx[gap_ok], order[gap_ok, :w])
        assert float((dd.double() - D.gather(1, idx)).abs().max()) < 1e-4
    i1, d1, m1 = eng.knn_rowmax(X, w, 40000, 333)
    i2, d2, m2 = eng.knn_rowmax(X, w, 39990, 1027)
    assert torch.equal(i1, i2[10:343]) and torch.equal(d1, d2[10:343]) and torch.equal(m1, m2[10:343])


def test_memory_100k_rows(eng):
    """N = 100k on one GPU, k = 10: the path's peak above the inputs stays below 1 GB (one dense N x N fp32 matrix
    would be 40 GB)"""
    from openibl_b200 import synth
    q, db, _ = synth.make_gallery(n_db=98000, n_q=2000, dim=256)
    q, db = q.cuda(), db.cuda()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ws0 = eng.rerank_workspace_bytes()
    from openibl_b200.evaluators import sharded_rerank_topk
    fd, fi = sharded_rerank_topk(q, db, 10, 0, db.shape[0], k1=20, k2=6, lambda_value=0.3)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    ws = max(eng.rerank_workspace_bytes(), ws0)
    assert peak + ws < 2 ** 30, (peak, ws)
    assert fi.shape == (2000, 10) and bool((fi >= 0).all())


def _bench(*extra):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "bench_rerank.py"), "--n-q", "300", "--n-db",
                          "2700", "--dim", "256", "--warmup", "0", *extra], capture_output=True, text=True,
                         timeout=900, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    return json.loads(out.stdout.strip().splitlines()[-1])


def test_world_size_independence():
    hashes = {w: _bench("--emulate-world", str(w))["topk_hash"] for w in (1, 3, 8)}
    assert len(set(hashes.values())) == 1, hashes
    if torch.cuda.device_count() >= 2:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
               "127.0.0.1", "--master-port", "29761", os.path.join(ROOT, "tools", "bench_rerank.py"), "--n-q", "300",
               "--n-db", "2700", "--dim", "256", "--warmup", "0"]
        out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
        assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
        line = [ln for ln in out.stdout.splitlines() if ln.startswith("{")][-1]
        assert json.loads(line)["topk_hash"] == hashes[1]


def test_evaluator_rerank_nms_matches_oracle():
    """Evaluator.evaluate(rerank=True, nms=True): k = 120 ranks per query, spatial NMS on the re-ranked list."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_gpu_e2e_api as E
    from oracle import ibl_oracle as O
    from openibl_b200.utils.rerank import re_ranking
    sys.path.insert(0, os.path.join(ROOT, "examples"))
    from eval_synthetic import SeededImages
    from openibl_b200 import datasets, models, synth
    ds = datasets.create("synthetic", None, n_db=E.N_DB, n_q=E.N_Q, seed=0)
    torch.manual_seed(0)
    base = models.create("vgg16", pretrained=False)
    pool = models.create("netvlad", dim=512)
    p = synth.make_netvlad_params(seed=0, sharp=True)
    pool.centroids.data.copy_(p["centroids"])
    pool.conv.weight.data.copy_(p["conv_weight"])
    sd = models.create("embednet", base, pool).state_dict()

    def feats(items):
        data = SeededImages(items, E.H, E.W)
        with torch.no_grad():
            return O.extract_descriptor(torch.stack([data[i][0] for i in range(len(items))]), sd, vlad=True)

    q, db = feats(ds.q_test), feats(ds.db_test)
    d = re_ranking(O.pairwise_distance(q, db).numpy(), O.pairwise_distance(q, q).numpy(),
                   O.pairwise_distance(db, db).numpy(), k1=10, k2=1, lambda_value=0.3)
    want = O.evaluate_all(d, ds.test_pos, [x[1] for x in ds.db_test], nms=True)
    got = E._run(1, 29773, extra=("--rerank", "--rr-topk", "10", "--lambda-value", "0.3", "--nms"))
    assert np.allclose(got, want, atol=2e-6), (got, want)


def test_evaluator_rerank_lambda0_matches_oracle():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_gpu_e2e_api import _oracle_recalls, _run
    want = _oracle_recalls(rerank=(10, 0.0))
    got = _run(1, 29771, extra=("--rerank", "--rr-topk", "10", "--lambda-value", "0.0"))
    assert np.allclose(got, want, atol=2e-6), (got, want)
    if torch.cuda.device_count() >= 2:
        want = _oracle_recalls(rerank=(10, 0.3))
        got = _run(2, 29772, extra=("--rerank", "--rr-topk", "10", "--lambda-value", "0.3"))
        assert np.allclose(got, want, atol=2e-6), (got, want)

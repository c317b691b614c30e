"""k-reciprocal re-ranking of dense distance matrices on the device (ibl_rerank_dense, Engine.rerank_dense), the route
re_ranking takes for host inputs -- the SFRS sampler refresh's call (examples/netvlad_img_sfrs.py:84) -- against the
unmodified reference function (tests/golden/rerank_sfrs.npz, tests/golden/rerank.npz) and the dense torch
restatement of openibl_b200/utils/rerank.py."""
import numpy as np
import pytest
import torch

from conftest import load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from openibl_b200.engine import Engine
    return Engine.get(0)


def _golden_cases():
    g = load_golden("rerank_sfrs")
    for name in ("sfrs", "k2", "asym", "tiny"):
        yield f"sfrs:{name}", g[f"{name}_qg"], g[f"{name}_qq"], g[f"{name}_gg"], g[f"{name}_final"], g[f"{name}_params"]
    g = load_golden("rerank")
    for name in "abc":
        yield f"rerank:{name}", g[f"{name}_qg"], g[f"{name}_qq"], g[f"{name}_gg"], g[f"{name}_final"], g[f"{name}_params"]


def test_reference_golden(eng):
    """Both entry points within 2e-6 of the reference's final matrix (the torch path's tolerance in test_host_cpu)."""
    from openibl_b200.utils.rerank import re_ranking
    for name, qg, qq, gg, want, (k1, k2, lam) in _golden_cases():
        k1, k2, lam = int(k1), int(k2), float(lam)
        got = eng.rerank_dense(*(torch.from_numpy(a).cuda() for a in (qg, qq, gg)), k1, k2, lam).cpu().numpy()
        assert got.shape == want.shape
        assert np.abs(got - want).max() <= 2e-6, (name, np.abs(got - want).max())
        host = re_ranking(qg, qq, gg, k1=k1, k2=k2, lambda_value=lam)
        assert isinstance(host, np.ndarray) and host.dtype == np.float32
        assert np.array_equal(host, got), name


def test_asymmetric_inputs_are_read_by_column(eng):
    """The reference's row i is column i of D: reading rows instead gives a different answer on the asym case."""
    g = load_golden("rerank_sfrs")
    qg, qq, gg, want = (torch.from_numpy(g[f"asym_{k}"]) for k in ("qg", "qq", "gg", "final"))
    k1, k2, lam = g["asym_params"]
    transposed = eng.rerank_dense(qg.cuda(), qq.t().contiguous().cuda(), gg.t().contiguous().cuda(), int(k1), int(k2),
                                  float(lam)).cpu()
    assert float((transposed - want).abs().max()) > 1e-4


def _separated(n_clusters, n_q, d, k1, seed):
    """test_gpu_rerank.py's margin-separated clusters (imported, not restated, where possible)"""
    from test_gpu_rerank import _separated as sep
    return sep(n_clusters, n_q, d, k1, seed)


def _dists(q, db):
    from test_gpu_rerank import _d64
    return _d64(q, db).float(), _d64(q, q).float(), _d64(db, db).float()


@pytest.mark.parametrize("n_clusters,n_q,d,k1,k2,lam", [
    (28, 63, 64, 20, 1, 0.1),              # the SFRS refresh's parameters
    (30, 33, 64, 10, 6, 0.3),
    (500, 500, 512, 10, 1, 0.1),           # m = 500, n = 5000
    (250, 500, 256, 20, 1, 0.3),           # m = 500, n = 4750
])
def test_agrees_with_torch_path(eng, n_clusters, n_q, d, k1, k2, lam):
    """Margin-separated data: values within 2e-6 of the torch restatement; with k2 = 1 (no exact ties from identical V
    rows) the same per-row ranking of the whole output."""
    from openibl_b200.utils.rerank import _re_ranking_torch
    q, db = _separated(n_clusters, n_q, d, k1, seed=n_clusters + k1)
    qg, qq, gg = (a.cuda() for a in _dists(q, db))
    got = eng.rerank_dense(qg, qq, gg, k1, k2, lam)
    want = _re_ranking_torch(qg, qq, gg, k1, k2, lam)
    assert float((got - want).abs().max()) <= 2e-6
    if k2 == 1:
        assert torch.equal(torch.argsort(got, dim=1, stable=True), torch.argsort(want, dim=1, stable=True))


def test_bit_identical_runs_and_edge_parameters(eng):
    from openibl_b200.utils.rerank import _re_ranking_torch, re_ranking
    q, db = _separated(30, 60, 64, 10, seed=3)
    qg, qq, gg = (a.cuda() for a in _dists(q, db))
    a = eng.rerank_dense(qg, qq, gg, 10, 1, 0.3)
    b = eng.rerank_dense(qg, qq, gg, 10, 1, 0.3)
    assert torch.equal(a, b)
    for k1, k2, lam in ((10, 1, 0.0), (10, 1, 1.0), (10, 11, 0.3), (10, 6, 0.0)):       # k2 = w = k1 + 1
        got = eng.rerank_dense(qg, qq, gg, k1, k2, lam)
        want = _re_ranking_torch(qg, qq, gg, k1, k2, lam)
        assert bool(torch.isfinite(got).all()) and float((got - want).abs().max()) <= 2e-6, (k1, k2, lam)
    # lambda = 1: the normalised original distances, exactly
    M = torch.cat([torch.cat([qq, qg], 1), torch.cat([qg.t(), gg], 1)], 0).pow(2).max(dim=0).values
    assert torch.equal(eng.rerank_dense(qg, qq, gg, 10, 1, 1.0), qg.pow(2) / M[:60, None])
    # m = 1
    got = eng.rerank_dense(qg[:1].contiguous(), qq[:1, :1].contiguous(), gg, 10, 1, 0.3)
    want = _re_ranking_torch(qg[:1], qq[:1, :1], gg, 10, 1, 0.3)
    assert got.shape == (1, db.shape[0]) and float((got - want).abs().max()) <= 2e-6
    # N < k1 + 1 on every route
    small = [x.cpu().numpy() for x in (qg[:2, :8], qq[:2, :2], gg[:8, :8])]
    with pytest.raises(ValueError):
        re_ranking(*small, k1=10, k2=1, lambda_value=0.3)
    with pytest.raises(ValueError):
        re_ranking(*(torch.from_numpy(x).cuda() for x in small), k1=10, k2=1, lambda_value=0.3)
    with pytest.raises(ValueError):
        eng.rerank_dense(qg[:2, :8].contiguous(), qq[:2, :2].contiguous(), gg[:8, :8].contiguous(), 10, 1, 0.3)
    # k1 = 130: neighbour lists wider than the kernels take; the host torch path answers
    q2, db2 = _separated(2, 70, 64, 130, seed=5)
    h = [x.numpy() for x in _dists(q2, db2)]
    got = re_ranking(*h, k1=130, k2=1, lambda_value=0.3)
    want = _re_ranking_torch(*(torch.from_numpy(x) for x in h), 130, 1, 0.3).numpy()
    assert np.array_equal(got, want)


def test_host_inputs_take_the_device_route(eng, monkeypatch):
    from openibl_b200.utils import rerank
    q, db = _separated(20, 40, 64, 10, seed=9)
    qg, qq, gg = _dists(q, db)
    want = eng.rerank_dense(qg.cuda(), qq.cuda(), gg.cuda(), 10, 1, 0.1).cpu()

    def refuse(*a, **k):
        raise AssertionError("host inputs reached the torch restatement")

    monkeypatch.setattr(rerank, "_re_ranking_torch", refuse)
    got = rerank.re_ranking(qg.numpy(), qq.numpy(), gg.numpy(), k1=10, k2=1, lambda_value=0.1)
    assert isinstance(got, np.ndarray) and np.array_equal(got, want.numpy())
    got_t = rerank.re_ranking(qg, qq, gg, k1=10, k2=1, lambda_value=0.1)        # CPU tensors in, CPU tensor out
    assert isinstance(got_t, torch.Tensor) and got_t.device.type == "cpu" and torch.equal(got_t, want)


def test_memory_at_pitts30k_train_shape(eng):
    """7,416 x 10,000: the device path's peak above its inputs and output stays below 1 GB (the dense torch path
    holds about 15 GB)."""
    from openibl_b200 import synth
    q, db, _ = synth.make_gallery(n_db=10000, n_q=7416, dim=256)
    q, db = q.cuda(), db.cuda()
    qg, qq, gg = eng.l2dist_dense(q, db), eng.l2dist_dense(q, q), eng.l2dist_dense(db, db)
    del q, db
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ws0 = eng.rerank_workspace_bytes()
    out = eng.rerank_dense(qg, qq, gg, 20, 1, 0.1)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base - out.numel() * 4
    ws = eng.rerank_workspace_bytes()
    assert peak + max(ws, ws0) < 2 ** 30, (peak, ws)
    assert out.shape == (7416, 10000) and bool(torch.isfinite(out).all())
    assert float(out.min()) >= 0.0 and float(out.max()) <= 1.0 + 1e-6


def test_sampler_difficult_positives_match_torch_path(eng):
    """DistributedRandomDiffTupleSampler.sort_gallery with the device route's Jaccard matrix deals the same tuples as
    with the torch path's, under the same RNG state."""
    import random
    from openibl_b200.utils.data.sampler import DistributedRandomDiffTupleSampler
    from openibl_b200.utils.rerank import _re_ranking_torch, re_ranking
    q, db = _separated(28, 63, 64, 20, seed=48)
    qg, qq, gg = _dists(q, db)
    m, n = qg.shape
    jac_dev = torch.from_numpy(re_ranking(qg.numpy(), qq.numpy(), gg.numpy(), k1=20, k2=1, lambda_value=0.1))
    jac_ref = _re_ranking_torch(qg.cuda(), qq.cuda(), gg.cuda(), 20, 1, 0.1).cpu()
    order = torch.argsort(qg, dim=1)
    pos = [order[i, :8].tolist() for i in range(m)]          # the 8 nearest gallery rows are "positives"
    neg = [order[i, :8].tolist() for i in range(m)]

    def tuples(jac):
        s = DistributedRandomDiffTupleSampler(list(range(m)), list(range(n)), pos, neg, pos_num=3, pos_pool=8,
                                              neg_num=4, neg_pool=100, num_replicas=1, rank=0)
        random.seed(7)
        s.sort_gallery(qg, jac, list(range(m)))
        return [t for t in iter(s)]

    assert tuples(jac_dev) == tuples(jac_ref)

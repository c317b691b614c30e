"""Searches over a prepared database (Engine.prepare_database / search_prepared, C ABI ibl_db_prepare / ibl_db_topk)
against ibl_l2dist_topk on the same rows: both are exact rankings under the same (distance, index) key and the same
exact fp32 arithmetic, so the results must agree bit for bit.  Paths of search_prepared (Engine.dist_path):

    0, 3  ibl_l2dist_topk itself   fp32 math mode, d % 64 != 0 (0); k > 12 (3, bf16x3 screening of the rows)
    1     single-pass fp16         m > 128, k <= 12, on the prepared plane
    4     streaming scan           m <= 128, k <= 12
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from openibl_b200.engine import Engine
    e = Engine.get(0)
    e.set_gemm_mode(1)
    yield e
    e.set_gemm_mode(1)


def expected_path(mode, m, d, k):
    if mode == 0 or d % 64 != 0:
        return 0
    if k > 12:
        return 3
    return 1 if m > 128 else 4


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


def same(eng, q, prep, k, idx_base=0, mode=1, what=""):
    """search_prepared == l2dist_topk bit for bit; returns (dist, idx, path of search_prepared, guard-listed)."""
    eng.set_gemm_mode(mode)
    try:
        wd, wi = eng.l2dist_topk(q, prep.rows, k, idx_base=idx_base)
        gd, gi = eng.search_prepared(q, prep, k, idx_base=idx_base)
        path, flagged = eng.dist_path(), eng.dist_flagged()
    finally:
        eng.set_gemm_mode(1)
    m, d = q.shape
    assert path == expected_path(mode, m, d, k), (what, path)
    assert torch.equal(gi, wi), f"{what}: indices differ (m={m}, n={prep.n}, d={d}, k={k})"
    assert torch.equal(gd, wd), f"{what}: distances differ (m={m}, n={prep.n}, d={d}, k={k})"
    return gd, gi, path, flagged


KS = (1, 10, 12, 13, 120, 128)


@pytest.mark.parametrize("n", [1, 16, 17, 129, 5000, 100000])
@pytest.mark.parametrize("m", [1, 3, 8, 9, 16, 17, 64, 65, 128, 129, 300])
def test_bit_identical_shapes(eng, m, n):
    """Query counts around every N of the streaming kernel and around the 128-query pass, database sizes around the
    16 survivors, the 128-row tile and the segment size of the row select; every k class; idx_base >= 2^31."""
    q, db = gallery(n, m, 512, seed=m * 7919 + n)
    prep = eng.prepare_database(db)
    seen = set()
    for k in KS:
        for idx_base in (0, 2 ** 31 + 7):
            seen.add(same(eng, q, prep, k, idx_base, what="shapes")[2])
    assert seen == ({1, 3} if m > 128 else {3, 4}), seen


@pytest.mark.parametrize("d", [64, 100, 512, 4096, 32768])
def test_bit_identical_dims(eng, d):
    """100: d % 64 != 0 goes to ibl_l2dist_topk; 32768: the raw-VLAD width; the fp32 math mode at every d."""
    for m, n in ((1, 5000), (9, 3000), (129, 1000), (300, 700)):
        q, db = gallery(n, m, d, seed=d + m)
        prep = eng.prepare_database(db)
        for k in (1, 10, 13, 128):
            same(eng, q, prep, k, 2 ** 31 + 7, what="dims")
            if m in (9, 300) and k in (10, 13):
                same(eng, q, prep, k, mode=0, what="fp32 mode")


def test_duplicates_keep_index_order(eng):
    """Identical rows give identical fp32 distances: the lower index comes first, on both prepared paths."""
    q, db = gallery(50, 160, 512, seed=4)
    prep = eng.prepare_database(torch.cat([db, db, db]).contiguous())
    for k in (3, 12, 13, 120):
        for qq in (q, q[:5].contiguous(), q[:100].contiguous()):
            _, ik, _, _ = same(eng, qq, prep, k, what="duplicates")
            assert (ik[:, 1] == ik[:, 0] + 50).all() and (ik[:, 2] == ik[:, 0] + 100).all()


@pytest.mark.parametrize("k", [10, 13, 120])
def test_ties_fire_the_guard(eng, k):
    """400 identical rows nearest to every query: no candidate list settles them, so the guard lists every query and
    the exact fallback ranks them, lowest indices first."""
    q, db = gallery(3000, 1, 512, seed=9)
    db[1000:1400] = q[0] + 0.01 * unit_rows(1, 512, gen(10))
    prep = eng.prepare_database(db)
    for m in (1, 64, 160):
        qq = q.repeat(m, 1).contiguous()
        _, ik, path, flagged = same(eng, qq, prep, k, what="400 ties")
        assert (ik == torch.arange(1000, 1000 + k, device="cuda")).all(), path
        assert flagged == m, (path, flagged)


@pytest.mark.parametrize("d", [512, 4096])
@pytest.mark.parametrize("m", [1, 8, 64, 128])
def test_screening_settles_retrieval_queries(eng, m, d):
    """On a retrieval-like gallery the fp16 screening decides almost every query by itself: the guard sends few to
    the exact fallback (a guard that listed everything would still give exact results, so bit-identity alone cannot
    show that the scan does the work)."""
    q, db = gallery(20000, m, d, seed=31 + m + d)
    prep = eng.prepare_database(db)
    for k in (1, 10):
        _, _, path, flagged = same(eng, q, prep, k, what="settled")
        assert path == 4
        assert 0 <= flagged <= max(1, m // 16), f"the guard listed {flagged} of {m} queries (d={d}, k={k})"


# ---- coherent rounding: the fp16 screening is wrong by far more than independent element errors would allow -------

def fp16_family(d, k):
    """q = 2^-7 on P = min(d, 4096) elements; the true nearest row X = 2^-7 (1 + 2^-11) there rounds onto q in fp16
    (exact distance P 2^-36, screened P 2^-24); k + 24 decoys, exact in fp16, lie between the two, so X falls out of
    every candidate list unless the guard catches it."""
    p = min(d, 4096)
    q = torch.zeros(1, d, device="cuda")
    q[:, :p] = 2.0 ** -7
    x = torch.zeros(1, d, device="cuda")
    x[:, :p] = 2.0 ** -7 * (1 + 2.0 ** -11)
    decoys = q.repeat(k + 24, 1)
    for j in range(k + 24):
        c = 1 + (j * 5) % (p // 32)
        cols = (torch.arange(c, device="cuda") + 13 * j) % p
        decoys[j, cols] -= 2.0 ** -10
    return q, x, decoys


@pytest.mark.parametrize("k", [1, 10, 120])
@pytest.mark.parametrize("d", [512, 4096, 32768])
@pytest.mark.parametrize("hidden", [False, True], ids=["near", "hidden"])
def test_coherent_rounding_ranks_exactly(eng, hidden, d, k):
    g = gen(d + k)
    q1, x, decoys = fp16_family(d, k)
    coherent = torch.cat([decoys[: len(decoys) // 2], x, decoys[len(decoys) // 2:]])
    filler = unit_rows(10000, d, g) if hidden else q1 + 0.01 * torch.randn(200, d, device="cuda", generator=g)
    n = len(filler) + len(coherent)
    pos = torch.randperm(n, device="cuda", generator=g)[: len(coherent)].sort().values
    db = torch.empty(n, d, device="cuda")
    keep = torch.ones(n, dtype=torch.bool, device="cuda")
    keep[pos] = False
    db[pos] = coherent
    db[keep] = filler
    ix = int(pos[len(decoys) // 2])
    prep = eng.prepare_database(db.contiguous())
    for m in (1, 64, 192):
        q = q1.repeat(m, 1).contiguous()
        dk, ik, path, flagged = same(eng, q, prep, k, what="coherent")
        assert (ik[:, 0] == ix).all(), f"path {path}: the true nearest row {ix} is not first"
        if path in (1, 4):        # fp16 screening: X is outside every candidate list, only the guard can find it
            assert flagged == m, f"path {path}: the guard listed {flagged} of {m} queries"
        exact = ((q[:1].double() - db[ix:ix + 1].double()) ** 2).sum()
        assert abs(float(dk[0, 0]) - float(exact)) <= 1e-6


# ---- no per-call database conversion --------------------------------------------------------------------------------

@pytest.mark.parametrize("m,k", [(1, 10), (64, 12), (128, 1), (300, 10)])
def test_launches_independent_of_n(eng, m, k):
    per_call = {}
    for n in (5000, 100000):
        q, db = gallery(n, m, 512, seed=n + m)
        prep = eng.prepare_database(db)
        eng.search_prepared(q, prep, k)
        c0 = eng.launch_count
        for _ in range(10):
            eng.search_prepared(q, prep, k)
        per_call[n] = (eng.launch_count - c0) / 10
    assert per_call[5000] == per_call[100000], per_call
    assert per_call[5000] == int(per_call[5000])


# ---- PlaceIndex on a synthetic Pittsburgh tree ----------------------------------------------------------------------

def _place_model():
    from openibl_b200 import models, synth
    torch.manual_seed(3)
    base = models.create("vgg16", pretrained=False)
    pool = models.create("netvlad", dim=base.feature_dim)
    p = synth.make_netvlad_params(seed=3, sharp=True)
    pool.centroids.data.copy_(p["centroids"])
    pool.conv.weight.data.copy_(p["conv_weight"])
    return models.create("embednet", base, pool).cuda()


def _loader(ds, items):
    from torch.utils.data import DataLoader
    from openibl_b200.utils.data import Preprocessor, get_transformer_test
    from openibl_b200.utils.data.sampler import DistributedSliceSampler
    pre = Preprocessor(items, root=ds.images_dir, transform=get_transformer_test(96, 128))
    return DataLoader(pre, batch_size=8, num_workers=2, sampler=DistributedSliceSampler(items, num_replicas=1, rank=0),
                      shuffle=False, pin_memory=True)


@pytest.fixture(scope="module")
def pitts(tmp_path_factory):
    from openibl_b200 import datasets
    from openibl_b200.evaluators import _extract_local
    from openibl_b200.pca import PCA
    root = tmp_path_factory.mktemp("place_index")
    datasets.write_synthetic_pitts_tree(str(root / "pitts"), scale="30k")
    ds = datasets.create("pitts", str(root / "pitts"), scale="30k", verbose=False)
    model = _place_model()
    feats, _ = _extract_local(model, _loader(ds, ds.db_test), vlad=True)
    pca = PCA(64, True, str(root / "pca_params.h5"))
    pca.train(feats)
    return root, ds, model, pca


@pytest.mark.parametrize("nms", [False, True])
def test_place_index_matches_evaluator(pitts, nms, tmp_path):
    import numpy as np
    from openibl_b200.evaluators import Evaluator, _extract_local, recalls_from_topk
    from openibl_b200.index import PlaceIndex
    root, ds, model, pca = pitts
    want = Evaluator(model).evaluate(_loader(ds, ds.q_test), None, ds.q_test, ds.db_test, ds.test_pos,
                                     gallery_loader=_loader(ds, ds.db_test), vlad=True, pca=pca, nms=nms)
    index = PlaceIndex.build(model, _loader(ds, ds.db_test), ds.db_test, pca=pca)
    x, _ = _extract_local(model, _loader(ds, ds.q_test), vlad=True, pca=pca)
    d, i = index.search(x, 10, nms=nms)
    if not nms:
        from openibl_b200.engine import Engine
        wd, wi = Engine.get(0).l2dist_topk(x, index.rows, 10)
        assert torch.equal(i, wi) and torch.equal(d, wd)
    got = recalls_from_topk(i.cpu().numpy(), ds.test_pos, ds.db_test, (1, 5, 10))
    assert np.array_equal(np.asarray(got), np.asarray(want)), (got, want)
    index.save(str(tmp_path))
    back = PlaceIndex.load(str(tmp_path), model=model)
    d2, i2 = back.search(x, 10, nms=nms)
    assert torch.equal(i, i2) and torch.equal(d, d2)
    imgs = next(iter(_loader(ds, ds.q_test)))[0]
    places = back.localize(imgs, k=10)
    plain = back.search(x, 10)[1][:len(imgs)].tolist()
    assert [[p[0] for p in row] for row in places] == [[ds.db_test[j][0] for j in r if j >= 0] for r in plain]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_place_index_two_ranks_one_rank(pitts, tmp_path):
    """Built on 2 ranks and loaded on 1, and the reverse (examples/localize.py under torchrun)."""
    import subprocess
    import sys
    root, ds, model, pca = pitts
    ckpt = tmp_path / "model.pth.tar"
    torch.save({"state_dict": model.state_dict()}, ckpt)
    outs = []
    for idx_dir, ranks in (("a", (2, 1)), ("b", (1, 2))):
        for r in ranks:
            cmd = [sys.executable] + (["-m", "torch.distributed.run", "--nproc-per-node", "2"] if r == 2 else [])
            cmd += [os.path.join(ROOT, "examples", "localize.py"), "--launcher", "pytorch" if r == 2 else "none",
                    *_example_args(root, ckpt, pca, tmp_path / idx_dir)]
            out = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
            assert out.returncode == 0, out.stderr[-3000:]
            outs.append((_recall_lines(out.stdout), open(tmp_path / idx_dir / "localize.csv").read()))
    assert all(o == outs[0] for o in outs)


import os  # noqa: E402
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _example_args(root, ckpt, pca, idx_dir):
    return ["-d", "pitts", "--scale", "30k", "--data-dir", str(root), "--resume", str(ckpt), "--vlad",
            "--pca-path", pca.pca_parameters_path, "--features", "64", "--index-dir", str(idx_dir),
            "--height", "96", "--width", "128", "--test-batch-size", "8", "-j", "2"]


def _recall_lines(stdout):
    return [ln.strip() for ln in stdout.splitlines() if ln.strip().startswith("top-")]


def test_localize_example_builds_then_loads(pitts, tmp_path):
    import subprocess
    import sys
    from openibl_b200.evaluators import Evaluator
    root, ds, model, pca = pitts
    want = Evaluator(model).evaluate(_loader(ds, ds.q_test), None, ds.q_test, ds.db_test, ds.test_pos,
                                     gallery_loader=_loader(ds, ds.db_test), vlad=True, pca=pca)
    want_lines = ["top-{:<4}{:12.1%}".format(kk, want[i]).strip() for i, kk in enumerate((1, 5, 10))]
    ckpt = tmp_path / "model.pth.tar"
    torch.save({"state_dict": model.state_dict()}, ckpt)
    cmd = [sys.executable, os.path.join(ROOT, "examples", "localize.py"),
           *_example_args(root, ckpt, pca, tmp_path / "index")]
    runs = []
    for _ in range(2):
        out = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
        assert out.returncode == 0, out.stderr[-3000:]
        runs.append((out.stdout, open(tmp_path / "index" / "localize.csv").read()))
    assert "built and saved" in runs[0][0] and "loaded the place index" in runs[1][0]
    assert _recall_lines(runs[0][0]) == want_lines, (runs[0][0], want_lines)
    assert _recall_lines(runs[1][0]) == want_lines
    assert runs[0][1] == runs[1][1]

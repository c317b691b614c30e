"""Host-side checks of the prepared-database search: the streaming scan kernel's SASS follows the issue discipline of
the other tensor-core kernels (wgmma fed by TMA, one elected lane issuing, no per-instruction issue loops)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "openibl_b200", "lib", "libiblb200.so")


@pytest.fixture(scope="module")
def scan_sass():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe) or not os.path.exists(LIB):
        pytest.skip("cuobjdump or the built library is missing")
    out = subprocess.run([exe, "-sass", LIB], capture_output=True, text=True, timeout=600).stdout
    counts, fn = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1) if "db_scan_dist_kernel" in m.group(1) else None
            if fn:
                counts[fn] = {}
            continue
        if fn is None:
            continue
        for op in ("HGMMA", "UTMALDG", "R2UR.BROADCAST", "BRA.U.ANY"):
            if re.search(r"\b" + re.escape(op), line):
                counts[fn][op] = counts[fn].get(op, 0) + 1
    return counts


def test_scan_kernel_runs_on_wgmma_and_tma(scan_sass):
    assert len(scan_sass) == 5, sorted(scan_sass)          # N = 8, 16, 32, 64, 128 queries per pass
    for k, c in scan_sass.items():
        assert c.get("HGMMA", 0) > 0 and c.get("UTMALDG", 0) > 0, (k, c)


def test_scan_kernel_has_no_per_instruction_issue_loops(scan_sass):
    for k, c in scan_sass.items():
        assert c.get("BRA.U.ANY", 0) == 0, (k, c)
        assert c.get("R2UR.BROADCAST", 0) <= 1, (k, c)


# ---- PlaceIndex: save format, re-slicing at other world sizes, errors (CPU stand-ins for the device search) ------

import json  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402


def _exact_search(q, rows, k, lo):
    """Exact CPU ranking by (fp64 distance, index) standing in for Engine.search_prepared."""
    d = torch.cdist(q.double(), rows.double()) ** 2
    m, n = d.shape
    dk = torch.full((m, k), float("inf"), dtype=torch.float32)
    ik = torch.full((m, k), -1, dtype=torch.int64)
    for r in range(m):
        order = sorted(range(n), key=lambda j: (float(d[r, j]), j))[:k]
        dk[r, :len(order)] = d[r, order].float()
        ik[r, :len(order)] = torch.tensor(order, dtype=torch.int64) + lo
    return dk, ik


def _merge(cd, ci, k):
    P, m, kk = cd.shape
    d = cd.permute(1, 0, 2).reshape(m, P * kk).numpy()
    i = ci.permute(1, 0, 2).reshape(m, P * kk).numpy()
    d = np.where(i < 0, np.inf, d)
    order = np.lexsort((i, d), axis=1)[:, :k]
    return torch.from_numpy(np.take_along_axis(d, order, 1)), torch.from_numpy(np.take_along_axis(i, order, 1))


def _use_cpu_standins(setattr_fn=setattr):
    from openibl_b200.index import PlaceIndex
    setattr_fn(PlaceIndex, "_prepare_fn", staticmethod(lambda rows: rows))
    setattr_fn(PlaceIndex, "_search_fn", staticmethod(_exact_search))
    setattr_fn(PlaceIndex, "_merge_fn", staticmethod(_merge))


@pytest.fixture
def standins(monkeypatch):
    _use_cpu_standins(monkeypatch.setattr)


def _fixture(n=37, dim=16, m=5):
    g = torch.Generator().manual_seed(n)
    db = torch.randn(n, dim, generator=g)
    q = db[:m] + 0.1 * torch.randn(m, dim, generator=g)
    gallery = [("db/%03d.jpg" % i, i // 2, 100.0 * i, 7.0 * i) for i in range(n)]
    return q, db, gallery


def _want(q, db, k):
    return _exact_search(q, db, k, 0)


def _save_or_load(rank, world, path, what):
    from openibl_b200.index import PlaceIndex
    from openibl_b200.utils.data.sampler import slice_bounds
    q, db, gallery = _fixture()
    if what == "save":
        lo, cnt, _ = slice_bounds(len(gallery), world, rank)
        idx = PlaceIndex(gallery, db[lo:lo + cnt].contiguous(), lo, len(gallery), db.shape[1], fingerprint="f" * 64)
        idx.save(path)
    else:
        idx = PlaceIndex.load(path, device=torch.device("cpu"))
    got = idx.search(q, 7)
    want = _want(q, db, 7)
    return bool(torch.equal(got[1], want[1]) and torch.equal(got[0], want[0]))


def _gloo_worker(rank, world, port, path, what, ret):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    _use_cpu_standins()
    try:
        ret[rank] = _save_or_load(rank, world, path, what)
    finally:
        dist.destroy_process_group()


def _run(world, path, what):
    if world == 1:                 # in this process: the test's fixture has installed the stand-ins
        return _save_or_load(0, 1, path, what)
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    with ctx.Manager() as mgr:
        ret = mgr.dict()
        port = 29400 + (os.getpid() + 37 * world + len(what)) % 150
        procs = [ctx.Process(target=_gloo_worker, args=(r, world, port, path, what, ret)) for r in range(world)]
        [p.start() for p in procs]
        [p.join(180) for p in procs]
        assert all(p.exitcode == 0 for p in procs)
        return all(ret.get(r) is True for r in range(world))


def test_save_format_round_trip(tmp_path, standins):
    from openibl_b200.index import PlaceIndex
    q, db, gallery = _fixture()
    idx = PlaceIndex(gallery, db, 0, len(gallery), db.shape[1], vlad=False, fingerprint="a" * 64)
    idx.save(str(tmp_path))
    meta = json.load(open(tmp_path / "index.json"))
    assert meta["format_version"] == 1 and meta["n"] == 37 and meta["dim"] == 16 and meta["vlad"] is False
    assert meta["model_sha256"] == "a" * 64 and meta["pca"] is None
    assert [tuple(it) for it in meta["gallery"]] == gallery
    assert meta["shards"] == [{"file": "rows_0.npy", "first": 0, "count": 37}]
    assert np.array_equal(np.load(tmp_path / "rows_0.npy"), db.numpy())
    back = PlaceIndex.load(str(tmp_path), device=torch.device("cpu"))
    assert back.gallery == gallery and torch.equal(back.rows, db) and back.vlad is False
    assert [torch.equal(a, b) for a, b in zip(back.search(q, 5), idx.search(q, 5))] == [True, True]


def test_reslice_2_to_1_and_1_to_3(tmp_path, standins):
    """Saved by 2 ranks, loaded by 1; saved by 1, loaded by 3 (gloo): the same exact ranking every time."""
    a, b = str(tmp_path / "w2"), str(tmp_path / "w1")
    assert _run(2, a, "save")
    assert sorted(os.listdir(a)) == ["index.json", "rows_0.npy", "rows_1.npy"]
    assert _run(1, a, "load")
    assert _run(1, b, "save")
    assert _run(3, b, "load")


def test_load_errors(tmp_path, standins):
    from openibl_b200.index import PlaceIndex, model_fingerprint
    q, db, gallery = _fixture()
    model = torch.nn.Linear(3, 2)
    path = str(tmp_path)
    PlaceIndex(gallery, db, 0, len(gallery), db.shape[1], fingerprint=model_fingerprint(model)).save(path)
    cpu = torch.device("cpu")
    PlaceIndex.load(path, model=model, device=cpu)                     # the same model loads
    wrapped = torch.nn.DataParallel(model)                             # `module.` names give the same fingerprint
    PlaceIndex.load(path, model=wrapped, device=cpu)
    with pytest.raises(ValueError, match="different model"):
        PlaceIndex.load(path, model=torch.nn.Linear(3, 2), device=cpu)
    np.save(os.path.join(path, "rows_0.npy"), db[:, :8].numpy())
    with pytest.raises(ValueError, match="rows_0.npy"):
        PlaceIndex.load(path, device=cpu)
    os.remove(os.path.join(path, "rows_0.npy"))
    with pytest.raises(FileNotFoundError, match="rows_0.npy"):
        PlaceIndex.load(path, device=cpu)

"""Tokyo 24/7 + Time Machine arranged from the raw dbStruct .mat files (`datasets.create('tokyo', root)`): the json
pair is byte-identical to the unmodified reference's on the seeded synthetic tree and takes the same values from
`random` (tests/golden/tokyo_arrange.npz, oracle/gen_golden_tokyo.py); an existing pair is left alone; under
torch.distributed only rank 0 writes; and the arrangement stays linear in the number of images."""
import json
import os
import random
import time

import numpy as np
import pytest

from conftest import load_golden

SPLITS = ("q_train", "db_train", "q_val", "db_val", "q_test", "db_test")


def _arrange(root, seed):
    from openibl_b200 import datasets
    random.seed(seed)
    ds = datasets.create("tokyo", root, verbose=False)
    return ds, random.random()


def _unragged(lens, flat):
    return np.split(flat, np.cumsum(lens)[:-1]) if len(lens) else []


@pytest.fixture(scope="module")
def golden_tree(tmp_path_factory):
    from openibl_b200.datasets import write_synthetic_tokyo_tree
    g = load_golden("tokyo_arrange")
    root = write_synthetic_tokyo_tree(str(tmp_path_factory.mktemp("tokyo") / "tokyo"), seed=int(g["tree_seed"]))
    return g, root


def test_arrangement_matches_reference_golden(golden_tree):
    g, root = golden_tree
    ds, nxt = _arrange(root, int(g["random_seed"]))
    for name in ("meta.json", "splits.json"):
        assert open(os.path.join(root, name), "rb").read() == g[name.replace(".", "_")].tobytes(), name
    assert nxt == float(g["next_random"])                        # the same number of draws from `random`
    for split in SPLITS:
        items = getattr(ds, split)
        assert [it[0] for it in items] == g[split + "_fname"].tolist(), split
        assert [it[1] for it in items] == g[split + "_pid"].tolist(), split
        assert np.array_equal(np.asarray([[it[2], it[3]] for it in items]).reshape(-1, 2), g[split + "_utm"]), split
    for k in ("train_pos", "val_pos", "test_pos"):
        want = _unragged(g[k + "_len"], g[k + "_flat"])
        got = getattr(ds, k)
        assert len(got) == len(want) and all(list(a) == b.tolist() for a, b in zip(got, want)), k


def test_synthetic_tree_exercises_every_arrangement_rule(golden_tree):
    """What the golden covers: Time Machine places with 1, 2 and 3 time stamps in both splits, a path listed twice,
    merged 24/7 query places, .png database files, landscape and portrait queries at several sizes, and a positive
    for every query."""
    from PIL import Image
    from openibl_b200.datasets.pitts import read_dbstruct
    g, root = golden_tree
    raw = os.path.join(root, "raw")
    for split in ("train", "val"):
        s = read_dbstruct(os.path.join(raw, "tokyoTM_%s.mat" % split), time_stamp=True)
        paths = s["q"] + s["db"]
        stamps = {}
        for p in paths:
            stamps.setdefault(p.split("/")[1], set()).add(p.split("/")[2])
        assert {len(v) for v in stamps.values()} == {1, 2, 3}, split
        assert len(paths) > len(set(paths)), split
    meta = json.loads(g["meta_json"].tobytes())
    splits = json.loads(g["splits_json"].tobytes())
    assert any(len(meta["identities"][p]) > 1 for p in splits["q_test"])                  # merged query places
    db = [f for p in splits["db_test"] for f in meta["identities"][p]]
    assert db and all(f.endswith(".png") and os.path.isfile(os.path.join(raw, f)) for f in db)
    shapes = {Image.open(os.path.join(raw, f)).size for p in splits["q_test"] for f in meta["identities"][p]}
    assert any(w > h for w, h in shapes) and any(h > w for w, h in shapes) and len(shapes) >= 4, shapes
    s = read_dbstruct(os.path.join(raw, "tokyo247.mat"))
    assert all(n.endswith(".jpg") for n in s["db"])
    n_q = {k: int(np.sum(g[k + "_len"] > 0)) for k in ("train_pos", "val_pos", "test_pos")}
    assert n_q["train_pos"] == len(g["q_train_pid"]) == len(g["db_train_pid"])             # no training query dropped
    assert n_q["val_pos"] == len(g["q_val_pid"]) and n_q["test_pos"] == len(g["q_test_pid"])


def test_missing_raw_raises_and_existing_json_pair_is_kept(tmp_path, golden_tree):
    import shutil
    from openibl_b200 import datasets
    with pytest.raises(RuntimeError, match="Dataset not found"):
        datasets.create("tokyo", str(tmp_path / "nothing"))
    g, src = golden_tree
    root = str(tmp_path / "tokyo")
    shutil.copytree(src, root)
    _arrange(root, 1)
    paths = [os.path.join(root, n) for n in ("meta.json", "splits.json")]
    past = time.time() - 3600
    for p in paths:
        os.utime(p, (past, past))
    before = [os.stat(p).st_mtime_ns for p in paths]
    random.seed(0)
    want = random.random()
    _, nxt = _arrange(root, 0)
    assert [os.stat(p).st_mtime_ns for p in paths] == before
    assert nxt == want                                    # nothing drawn when the pair already exists


def _gloo_worker(rank, world, port, root, ret):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import openibl_b200.utils.serialization as S
        import openibl_b200.datasets.tokyo as T
        written = []
        real = S.write_json

        def spy(obj, fpath):
            written.append(os.path.basename(fpath))
            real(obj, fpath)
        T.write_json = spy
        if rank == 1:
            time.sleep(1.0)                        # rank 0 finishes its arrangement long before rank 1 starts
        ds, nxt = _arrange(root, 43)
        ret[rank] = dict(written=written, next=nxt,
                         splits={k: [tuple(it) for it in getattr(ds, k)] for k in SPLITS},
                         pos=[list(map(int, p)) for p in ds.test_pos + ds.val_pos + ds.train_pos])
    finally:
        dist.destroy_process_group()


def test_world2_gloo_only_rank0_writes_and_ranks_agree(tmp_path):
    import torch.multiprocessing as mp
    from openibl_b200.datasets import write_synthetic_tokyo_tree
    g = load_golden("tokyo_arrange")
    root = write_synthetic_tokyo_tree(str(tmp_path / "tokyo"), seed=int(g["tree_seed"]))
    ctx = mp.get_context("spawn")
    with ctx.Manager() as mgr:
        ret = mgr.dict()
        port = 29400 + os.getpid() % 200
        procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, root, ret)) for r in range(2)]
        [p.start() for p in procs]
        [p.join(180) for p in procs]
        assert all(p.exitcode == 0 for p in procs)
        r0, r1 = dict(ret[0]), dict(ret[1])
    assert r0["written"] == ["meta.json", "splits.json"] and r1["written"] == []
    assert r0["splits"] == r1["splits"] and r0["pos"] == r1["pos"]
    assert r0["next"] == r1["next"] == float(g["next_random"])   # both ranks arranged and drew alike
    for name in ("meta.json", "splits.json"):
        assert open(os.path.join(root, name), "rb").read() == g[name.replace(".", "_")].tobytes(), name


def _write_large_tm(raw, n_places, stamps, views):
    """Only the .mat files: the arrangement reads no image.  n_places x stamps x views images per split."""
    from scipy.io import savemat
    for split in ("train", "val"):
        names = ["%02d/%s%06d/%d/%d.jpg" % (p % 100, split, p, t, v)
                 for p in range(n_places) for t in range(stamps) for v in range(views)]
        utm = np.asarray([[1000.0 * (p % 300), 1000.0 * (p // 300)] for p in range(n_places)
                          for _ in range(stamps * views)]).T
        half = len(names) // 2
        cell = lambda xs: np.array([[n] for n in xs], dtype=object)
        st = {"whichSet": split, "dbImageFns": cell(names[half:]), "utmDb": utm[:, half:], "dbTimeStamp": np.zeros((1, 1)),
              "qImageFns": cell(names[:half]), "utmQ": utm[:, :half], "qTimeStamp": np.zeros((1, 1)),
              "numImages": 0.0, "numQueries": 0.0}
        savemat(os.path.join(raw, "tokyoTM_%s.mat" % split), {"dbStruct": st})
    cell = lambda xs: np.array([[n] for n in xs], dtype=object)
    savemat(os.path.join(raw, "tokyo247.mat"), {"dbStruct": {
        "whichSet": "test", "dbImageFns": cell(["00/0.jpg"]), "utmDb": np.zeros((2, 1)),
        "qImageFns": cell(["0.jpg"]), "utmQ": np.ones((2, 1)), "numImages": 1.0, "numQueries": 1.0}})


def test_arrangement_is_linear_in_the_number_of_images(tmp_path):
    """10 000 Time Machine places of 2 time stamps x 2 views per split, 80 000 paths: list membership tests
    (`p in train_pids` over the place ids) would make this quadratic in the number of places; with sets it arranges in
    about 1.1 s on one core of a current x86 server CPU, most of it in loadmat and json.dump."""
    from openibl_b200.datasets.tokyo import Tokyo
    root = str(tmp_path / "tokyo")
    os.makedirs(os.path.join(root, "raw"))
    _write_large_tm(os.path.join(root, "raw"), n_places=10000, stamps=2, views=2)
    ds = Tokyo.__new__(Tokyo)
    ds.root = root
    random.seed(0)
    t0 = time.perf_counter()
    ds.arrange()
    dt = time.perf_counter() - t0
    splits = json.load(open(os.path.join(root, "splits.json")))
    assert len(splits["q_train"]) == 20000 and len(splits["q_val"]) == 10000 and len(splits["db_val"]) == 10000
    assert dt < 10.0, dt

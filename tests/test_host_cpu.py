"""CPU-side tests: C-ABI library loads and exports every declared symbol, the host mirror keeps the
reference's plugin API (config 1 plumbing), recall logic matches the oracle, the N>1 host logic
works under gloo.  No GPU compute here."""
import os
import re
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden
from oracle import ibl_oracle as O
from openibl_b200 import synth


def test_cabi_exports_every_declared_symbol():
    from openibl_b200 import _cabi
    lib = _cabi.load()
    header = open(os.path.join(ROOT, "include", "iblb200.h")).read()
    declared = set(re.findall(r"^(?:int|const char\*)\s+(ibl_\w+)\s*\(", header, flags=re.M))
    assert len(declared) >= 25
    assert declared == set(_cabi.SIGNATURES), declared ^ set(_cabi.SIGNATURES)
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.ibl_abi_version() == 1
    assert lib.ibl_status_string(4).decode().startswith("no usable sm_90")


@pytest.mark.skipif(torch.cuda.is_available(), reason="CPU-only behaviour")
def test_no_cpu_fallback_engine_create_fails_loudly():
    import ctypes
    from openibl_b200 import _cabi
    lib = _cabi.load()
    h = ctypes.c_void_p()
    st = lib.ibl_engine_create(0, ctypes.byref(h))
    assert st == 4 and not h.value            # IBL_ERR_NO_DEVICE
    assert b"no CPU fallback" in lib.ibl_last_error()
    from openibl_b200.engine import Engine
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        Engine.get(0)


def test_config1_plumbing_hubconf_on_cpu():
    """BASELINE configs[0]: hubconf.vgg16_netvlad(pretrained=False) builds on CPU with the reference's
    30 state-dict keys and shapes; its forward is GPU-only and says so."""
    sys.path.insert(0, ROOT)
    import hubconf
    model = hubconf.vgg16_netvlad(pretrained=False)
    sd = model.state_dict()
    want = synth.make_state_dict(seed=0, with_pca=True)
    assert list(sd.keys()) == list(want.keys())
    for k in sd:
        assert tuple(sd[k].shape) == tuple(want[k].shape), k
    assert sum(v.numel() for v in sd.values()) == 149002048
    model.load_state_dict(want)
    assert model.base_model.feature_dim == 512
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        model.eval()(torch.randn(1, 3, 480, 640))


def test_models_factory_contract():
    from ibl import models
    assert models.names() == ["embednet", "embednetpca", "embedregionnet", "netvlad", "vgg16"]
    with pytest.raises(KeyError):
        models.create("resnet50")
    base = models.create("vgg16", pretrained=False, cut_at_pooling=True)
    nv = models.create("netvlad", num_clusters=64, dim=512, alpha=100.0, normalize_input=True)
    assert nv.conv.weight.shape == (64, 512, 1, 1) and nv.centroids.shape == (64, 512)
    emb = models.create("embedregionnet", base, nv, tuple_size=4)
    assert emb.tuple_size == 4
    # DDP-style prefixed checkpoints load through copy_state_dict (examples/test.py:97-99)
    from ibl.utils.serialization import copy_state_dict
    src = {"module." + k: v for k, v in synth.make_state_dict(seed=3, with_pca=False).items()}
    wrapped = torch.nn.Sequential()
    wrapped.add_module("module", models.create("embednet", models.create("vgg16", pretrained=False), nv))
    copy_state_dict(src, wrapped)
    assert torch.equal(wrapped.state_dict()["module.net_vlad.centroids"], src["module.net_vlad.centroids"])


def test_netvlad_init_params_matches_reference_golden():
    g = load_golden("netvlad_unit")
    from ibl import models
    nv = models.create("netvlad", dim=512)
    gg = synth._gen(3 + 1000)
    clsts = torch.randn(64, 512, generator=gg)
    clsts = clsts / clsts.norm(dim=1, keepdim=True)
    desc = torch.randn(5000, 512, generator=gg)
    desc = desc / desc.norm(dim=1, keepdim=True)
    nv.clsts = clsts.numpy().astype(np.float32)
    nv.traindescs = desc.numpy().astype(np.float32)
    nv._init_params()
    assert abs(nv.alpha - float(g["alpha"])) < 1e-4 * float(g["alpha"])


def test_recalls_from_topk_matches_reference_golden():
    from openibl_b200.evaluators import recalls_from_topk, spatial_nms
    g = load_golden("retrieval")
    q, db, gt = synth.make_gallery(n_db=1500, n_q=300, dim=512, sigma=0.28)
    gallery = [("d%05d" % i, i // 3, 0.0, 0.0) for i in range(1500)]
    gt_list = [np.array([int(t)]) for t in gt]
    d = O.pairwise_distance(q, db).numpy()
    _, idx120 = O.topk_from_distmat(d, 120)
    assert np.array_equal(recalls_from_topk(idx120[:, :10], gt_list, gallery), g["recalls"])
    assert np.array_equal(recalls_from_topk(idx120, gt_list, gallery, nms=True), g["recalls_nms"])
    pids = [p[1] for p in gallery]
    assert spatial_nms(idx120[0].tolist(), pids, 120) == O.spatial_nms(idx120[0].tolist(), pids, 120)


def test_slice_sampler_matches_reference_semantics():
    from ibl.utils.data.sampler import DistributedSliceSampler, slice_bounds
    data = list(range(10))
    got = [list(DistributedSliceSampler(data, num_replicas=4, rank=r)) for r in range(4)]
    # reference sampler.py:208-219: ceil(10/4)=3 per rank, tail wraps to the head
    assert got == [[0, 1, 2], [3, 4, 5], [6, 7, 8], [9, 0, 1]]
    assert [slice_bounds(10, 4, r) for r in range(4)] == [(0, 3, 3), (3, 3, 3), (6, 3, 3), (9, 1, 3)]
    assert len(DistributedSliceSampler(data, num_replicas=4, rank=3)) == 3


def _gloo_worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from openibl_b200.evaluators import sharded_topk
        from openibl_b200.utils.data.sampler import slice_bounds
        q, db, gt = synth.make_gallery(n_db=1001, n_q=37, dim=64, sigma=0.5)
        lo, cnt, per = slice_bounds(db.shape[0], world, rank)
        shard = torch.zeros(per, db.shape[1])
        shard[:cnt] = db[lo:lo + cnt]

        def rank_fn(qq, dd, k, idx_base, n_valid):     # oracle stands in for the CUDA kernel
            d = O.pairwise_distance(qq, dd[:n_valid]).numpy()
            dk, ik = O.topk_from_distmat(d, min(k, n_valid))
            pad = k - dk.shape[1]
            dk = np.pad(dk, ((0, 0), (0, pad)), constant_values=np.inf)
            ik = np.pad(ik + idx_base, ((0, 0), (0, pad)), constant_values=-1)
            return torch.from_numpy(dk), torch.from_numpy(ik)

        def merge_fn(cd, ci, k):
            P, m, kk = cd.shape
            d = cd.permute(1, 0, 2).reshape(m, P * kk).numpy()
            i = ci.permute(1, 0, 2).reshape(m, P * kk).numpy()
            d = np.where(i < 0, np.inf, d)
            order = np.lexsort((i, d), axis=1)[:, :k]
            return torch.from_numpy(np.take_along_axis(d, order, 1)), torch.from_numpy(np.take_along_axis(i, order, 1))

        dk, ik = sharded_topk(q, shard, 10, idx_base=lo, n_valid=cnt, _rank_fn=rank_fn, _merge_fn=merge_fn)
        full = O.pairwise_distance(q, db).numpy()
        wd, wi = O.topk_from_distmat(full, 10)
        ok = bool(np.array_equal(ik.numpy(), wi) and np.allclose(dk.numpy(), wd, atol=1e-6))

        # Evaluator.evaluate end to end (shard-resident path): fake descriptors keyed by file name stand in
        # for the CUDA forward; loaders are DistributedSliceSampler slices like examples/test.py:38-54
        import openibl_b200.evaluators as E
        from torch.utils.data import DataLoader
        from openibl_b200.utils.data.sampler import DistributedSliceSampler
        query = [("q/%04d.jpg" % i, 2000 + i, 0.0, 0.0) for i in range(q.shape[0])]
        gallery = [("db/%04d.jpg" % i, i // 2, 0.0, 0.0) for i in range(db.shape[0])]
        table = {f: r for (f, _, _, _), r in zip(query + gallery, torch.cat([q, db]))}

        class Items(torch.utils.data.Dataset):
            def __init__(self, items): self.items = items
            def __len__(self): return len(self.items)
            def __getitem__(self, i):
                f, pid, x, y = self.items[i]
                return torch.zeros(1), f, pid, x, y

        seen = []
        def fake_feature(model, inputs, vlad=True, gpu=None):
            names = seen.pop(0)
            return torch.stack([table[n] for n in names])

        def loader(items, sampler=None):
            dl = DataLoader(Items(items), batch_size=8, sampler=sampler or DistributedSliceSampler(items), shuffle=False)
            class Spy:                      # records the batch's file names for the fake forward
                def __iter__(s):
                    for b in dl:
                        seen.append(list(b[1]))
                        yield b
                def __len__(s): return len(dl)
            return Spy()

        E.extract_cnn_feature = fake_feature
        ev = E.Evaluator(torch.nn.Identity())
        E.Evaluator._rank_fn, E.Evaluator._merge_fn = staticmethod(rank_fn), staticmethod(merge_fn)
        gt_list = [np.array([int(t)]) for t in gt]
        want = O.recalls_from_ranking(O.topk_from_distmat(full, 10)[1], gt_list, [g[1] for g in gallery])
        got = ev.evaluate(loader(query), None, query, gallery, gt_list, gallery_loader=loader(gallery))
        ok = ok and np.array_equal(got, want) and ev.last_stats.get("d2h_descriptor_bytes") == 0
        want_nms = O.recalls_from_ranking(O.topk_from_distmat(full, 120)[1], gt_list, [g[1] for g in gallery], nms=True)
        got_nms = ev.evaluate(loader(query), None, query, gallery, gt_list, gallery_loader=loader(gallery), nms=True)
        ok = ok and np.array_equal(got_nms, want_nms)
        # a loader that does NOT follow the slice layout (every rank sees everything) takes the by-name path
        dataset = sorted(query + gallery)
        from torch.utils.data.sampler import SequentialSampler
        got2 = ev.evaluate(loader(dataset, SequentialSampler(dataset)), dataset, query, gallery, gt_list)
        ok = ok and np.array_equal(got2, want)
        rev = list(reversed(gallery))
        got3 = ev.evaluate(loader(query), None, query, gallery, gt_list,
                           gallery_loader=loader(rev, DistributedSliceSampler(rev)))
        ok = ok and np.array_equal(got3, want)
        ret[rank] = ok
    finally:
        dist.destroy_process_group()


def test_sharded_topk_and_evaluator_world2_gloo():
    """N>1 host logic on CPU: slice the database like DistributedSliceSampler, all-gather the per-shard
    candidates (packed fp32 + int32) over gloo, merge; must equal the single-process oracle ranking.  Then
    Evaluator.evaluate at world size 2 (shard-resident path, nms path, by-name fallback paths) against the
    oracle's recalls, with the kernels replaced by the oracle."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    with ctx.Manager() as mgr:
        ret = mgr.dict()
        port = 29600 + os.getpid() % 200
        procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, ret)) for r in range(2)]
        [p.start() for p in procs]
        [p.join(180) for p in procs]
        assert all(p.exitcode == 0 for p in procs)
        assert ret.get(0) is True and ret.get(1) is True


def _pca_fixture(n_pts, n_dims, seed):
    g = torch.Generator().manual_seed(seed)
    basis = torch.randn(n_dims, n_dims, generator=g)
    scale = torch.logspace(0, -2, n_dims)
    return (torch.randn(n_pts, n_dims, generator=g) * scale) @ basis + torch.randn(n_dims, generator=g)


def test_pca_parameter_store_roundtrip_and_load_contract(tmp_path):
    """The h5-free parameter store of PCA (reference pca.py:79-84 writes {U, lams, mu, Utmu} to h5): what train()
    saves is what load() reads; parameters here come from the oracle's restatement of relja_PCA (the fit itself runs
    on the GPU engine and is tested there: test_pca_fit_load_infer_roundtrip_vs_oracle)."""
    from openibl_b200.pca import PCA
    for n_pts, n_dims, P in ((300, 64, 16), (40, 96, 12)):
        x = _pca_fixture(n_pts, n_dims, seed=n_pts)
        U, lams, mu, Utmu = O.pca_train(x.clone(), n_components=P)
        path = str(tmp_path / f"pca_{n_pts}.h5")
        pca = PCA(pca_n_components=P, pca_whitening=True, pca_parameters_path=path)
        pca._save(U=U, lams=lams, mu=mu, Utmu=Utmu)
        got = pca._read()
        for k, v in (("U", U), ("lams", lams), ("mu", mu), ("Utmu", Utmu)):
            np.testing.assert_array_equal(got[k], v)
        assert os.path.isfile(path)      # examples/test.py:111 checks osp.isfile(pca_parameters_path)
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            PCA(4, True, str(tmp_path / "x.h5")).train(torch.randn(10, 8))


def test_rerank_matches_reference_golden():
    """k-reciprocal re-ranking (ibl/utils/rerank.py:32-100, called from evaluators.py:194-199) restated as dense
    set algebra: same distances as the unmodified reference function on three seeded cases (k2 = 1 as the
    evaluator calls it, and k2 = 3 with query expansion)."""
    from ibl.utils.rerank import re_ranking
    g = load_golden("rerank")
    for name in "abc":
        k1, k2, lam = g[f"{name}_params"]
        out = re_ranking(g[f"{name}_qg"], g[f"{name}_qq"], g[f"{name}_gg"], k1=int(k1), k2=int(k2), lambda_value=float(lam))
        assert isinstance(out, np.ndarray) and out.shape == g[f"{name}_final"].shape
        np.testing.assert_allclose(out, g[f"{name}_final"], atol=2e-6, rtol=0)
        t = re_ranking(torch.from_numpy(g[f"{name}_qg"]), torch.from_numpy(g[f"{name}_qq"]), torch.from_numpy(g[f"{name}_gg"]),
                       k1=int(k1), k2=int(k2), lambda_value=float(lam))
        assert torch.is_tensor(t) and np.allclose(t.numpy(), out)


def test_sfrs_loss_algebra_matches_reference_golden():
    """SFRSTrainer._get_loss / _get_hard_loss (trainers.py:261-320) against the unmodified reference trainer on random
    unit-norm region descriptors (tests/golden/sfrs_step.npz, oracle/gen_golden_sfrs.py)."""
    from ibl.trainers import SFRSTrainer
    g = load_golden("sfrs_step")
    tr = SFRSTrainer(None, None, margin=0.1, neg_num=3, gpu=None, temp=[0.07, 0.07])
    a, p, n = (torch.from_numpy(g[k]) for k in ("u_anchors", "u_positives", "u_negatives"))
    for lt in ("triplet", "sare_joint", "sare_ind"):
        assert abs(tr._get_loss(a, p, n, 4, lt).item() - float(g[f"u_loss_{lt}"])) < 2e-6, lt
    got = tr._get_hard_loss(a[0], p[0], torch.from_numpy(g["u_hard_negatives"]), torch.from_numpy(g["u_hard_scores"]), "sare_ind")
    assert abs(got.item() - float(g["u_hard_loss"])) < 2e-6
    with pytest.raises(ValueError):
        tr._get_loss(a, p, n, 4, "nope")


def _sampler_fixture():
    g = load_golden("sampler")
    NQ, NG = g["dist"].shape
    q = [("q%03d" % i, i, 0.0, 0.0) for i in range(NQ)]
    gal = [("g%03d" % i, 1000 + i, 0.0, 0.0) for i in range(NG)]
    pos_l = [p.tolist() for p in g["pos"]]
    neg_l = [sorted(set(n.tolist())) for n in g["neg"]]
    return g, q, gal, pos_l, neg_l, list(range(3, NQ, 2))


def test_tuple_samplers_yield_reference_tuples_given_the_reference_ranking():
    """DistributedRandomTupleSampler / DistributedRandomDiffTupleSampler (sampler.py:15-192): with the same ranking
    and the same `random` state the host logic yields exactly the reference's tuples, over two epochs (cached hard
    negatives) and two ranks.  The ranking itself comes from the device argsort on the GPU (test_gpu_parity)."""
    import random
    from ibl.utils.data.sampler import DistributedRandomTupleSampler, DistributedRandomDiffTupleSampler
    g, q, gal, pos_l, neg_l, sub = _sampler_fixture()
    for name, cls, kw in (("tuple", DistributedRandomTupleSampler, dict(neg_num=4, neg_pool=30)),
                          ("diff", DistributedRandomDiffTupleSampler, dict(pos_num=3, pos_pool=5, neg_num=4, neg_pool=30))):
        for rank in (0, 1):
            s = cls(q, gal, pos_l, neg_l, num_replicas=2, rank=rank, **kw)
            random.seed(11 + rank)
            s.sort_idx, s.sub_set, s.sub_length = torch.from_numpy(g["sort_idx"]), sub, len(sub)
            s._resize()
            if name == "diff":
                s.distmat_jac = torch.from_numpy(g["jac"])
            assert len(s) == int(g[f"{name}_len"])
            for ep in (0, 1):
                got = np.asarray([r + [-1] * (9 - len(r)) for r in iter(s)], dtype=np.int64)   # ragged rows padded with -1
                assert np.array_equal(got, g[f"{name}_r{rank}_e{ep}"]), (name, rank, ep)


def test_distance_screening_selection_model_keeps_the_true_top16():
    """Model check of the selection logic of gemm2_f16_top16_kernel's epilogue (tc_dist1.cu): per work item a sorted
    top-16, a threshold that is only refreshed at merges, a 32-slot pending list flushed when it could overflow within
    the next 16 columns, and a per-query gate shared between concurrently running items through atomicMin with
    arbitrarily STALE reads.  Whatever the interleaving, the union of the items' lists must contain the true 16
    smallest screened distances of the row (the guard of dist_finish_kernel assumes exactly that)."""
    import numpy as np
    rng = np.random.RandomState(11)
    PEND, TILE = 32, 256

    def run_row(vals, n_items, order_seed, adversarial):
        n = len(vals)
        per = -(-n // (n_items * TILE)) * TILE
        items = [dict(lo=i * per, hi=min(n, (i + 1) * per), pos=i * per, td=[np.inf] * 16, ti=[-1] * 16, thr=np.inf,
                      pend=[]) for i in range(n_items)]
        gate_hist = [np.inf]                                  # every value the gate ever had: a reader may see any of them
        sched = np.random.RandomState(order_seed)

        def merge(it):
            for d, c in it["pend"]:
                if d < it["td"][15]:
                    p = sum(1 for t in it["td"] if t <= d)
                    it["td"].insert(p, d); it["ti"].insert(p, c)
                    it["td"].pop(); it["ti"].pop()
            it["pend"] = []

        live = [it for it in items if it["pos"] < it["hi"]]
        while live:
            it = live[sched.randint(len(live))]
            seen = gate_hist[sched.randint(len(gate_hist))] if adversarial else gate_hist[-1]
            it["thr"] = min(it["thr"], seen)                  # stale or fresh gate read at the start of a tile
            end = min(it["hi"], it["pos"] + TILE)
            for g0 in range(it["pos"], end, 16):
                if len(it["pend"]) > PEND - 16:
                    merge(it)
                    it["thr"] = min(it["thr"], it["td"][15])
                for c in range(g0, min(end, g0 + 16)):
                    if vals[c] < it["thr"]:
                        it["pend"].append((vals[c], c))
                assert len(it["pend"]) <= PEND
            merge(it)
            if it["td"][15] < it["thr"]:
                it["thr"] = it["td"][15]
                gate_hist.append(min(gate_hist[-1], it["thr"]))
            it["pos"] = end
            live = [x for x in items if x["pos"] < x["hi"]]
        got = sorted(d for it in items for d in it["td"] if np.isfinite(d))[:16]
        return np.array(got)

    for trial in range(40):
        n = int(rng.choice([300, 1000, 4096, 10000]))
        kind = trial % 4
        if kind == 0:
            vals = rng.rand(n)
        elif kind == 1:
            vals = np.sort(rng.rand(n))[::-1].copy()          # descending: every column beats the running 16th best
        elif kind == 2:
            vals = np.round(rng.rand(n), 2)                   # heavy ties, also at the threshold
        else:
            vals = np.abs(rng.randn(n)) * (1 + (np.arange(n) % 7 == 0) * -0.9)
        vals = vals.astype(np.float32)
        want = np.sort(vals)[:16]
        for n_items in (1, 3, 8):
            got = run_row(vals, n_items, order_seed=trial * 10 + n_items, adversarial=True)
            # A candidate is dropped only against a gate that is some item's 16th best, i.e. that item holds 16 values
            # <= the gate -- so every dropped value is >= the merged 16th best and the merged VALUES are exactly the 16
            # smallest (with ties at the 16th place, which copy survives is arbitrary; the indices are not compared).
            assert np.array_equal(got, want[: len(got)]) and len(got) == min(16, n), (trial, n_items, got, want)

"""Tokyo 24/7 + Time Machine end to end on a synthetic tree that `datasets.create('tokyo', root)` arranges from its raw
dbStruct .mat files (`write_synthetic_tokyo_tree`):

* the reference's examples/test.py (byte-identical, tests/fixtures/reference_examples_test.py.txt) with `-d tokyo`
  under torch.distributed.run with one and with two processes: batch-1 `Resize(640)`-style queries, Recall@N with
  spatial NMS, PCA fitted on the synthetic Pittsburgh tree as the script always does; the printed recalls equal the
  CPU oracle's on the same images, checkpoint and PCA fit;
* the reference's examples/cluster.py and examples/netvlad_img.py (byte-identical, tests/golden/) with `-d tokyo`: one
  short epoch on Time Machine tuples (q_train == db_train), validation on q_val / db_val, a checkpoint written; and the
  first training step -- the model the driver starts from, the first tuple its sampler deals after seeding `random`
  -- gives the CPU oracle's loss on the engine;
* Tokyo 24/7 queries of mixed orientation and size decoded on the device with the `tokyo=True` transform: the
  features equal the host transform's bit for bit, and no file reaches the host decoder."""
import hashlib
import os
import random
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN, ROOT
from openibl_b200 import synth

pytestmark = pytest.mark.gpu

TEST_PY = os.path.join(ROOT, "tests", "fixtures", "reference_examples_test.py.txt")
TEST_PY_SHA256 = "23a3d57dc1af659c8b9aab1acb6d75c2b4d75b8312e4c52f3d91b8de342e70c0"
SCRIPTS = {"cluster": "785c1fcf8219c58fdbbb4be5cc7df7013174162b18fe3db7853256f1b0a68452",
           "netvlad_img": "9f2c21800b4cadc563d4e3072dc5b74c193f3133070574391d2429c7e9adbbd5"}
H, W, FEATURES = 96, 128, 32
RH, RW = 160, 256                 # conv5 map 10 x 16 = 160 locations >= the 100 cluster.py samples per image
TM_TRAIN_PLACES = 132             # 1 + p % 3 time stamps x 2 views: 528 training images >= the 500 cluster.py samples
TWO_GPUS = torch.cuda.is_available() and torch.cuda.device_count() >= 2
MARGIN = 0.1 ** 0.5


def _checkpoint(path):
    from ibl import models
    from ibl.utils.serialization import save_checkpoint
    torch.manual_seed(3)
    base = models.create("vgg16", pretrained=False)
    pool = models.create("netvlad", dim=base.feature_dim)
    p = synth.make_netvlad_params(seed=3, sharp=True)
    pool.centroids.data.copy_(p["centroids"])
    pool.conv.weight.data.copy_(p["conv_weight"])
    model = models.create("embednet", base, pool)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    save_checkpoint({"state_dict": {"module." + k: v for k, v in sd.items()}, "epoch": 3, "best_recall5": 0.5},
                    False, fpath=path)
    return sd


def _oracle_feats(ds, items, tf, sd, pca=None):
    """One image at a time: Tokyo queries keep their aspect ratio, so their sizes differ."""
    from ibl.utils.data.preprocessor import Preprocessor
    from oracle import ibl_oracle as O
    pre = Preprocessor(items, root=ds.images_dir, transform=tf)
    with torch.no_grad():
        out = torch.cat([O.extract_descriptor(pre[i][0][None], sd, vlad=True) for i in range(len(items))])
    return out if pca is None else O.pca_whiten(out, *pca)


# ---- examples/test.py -d tokyo ------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def eval_setup(tmp_path_factory):
    """The raw trees (a fresh copy per run, so that every run arranges Tokyo itself), the checkpoint, and the CPU
    oracle's Recall@1/5/10 with spatial NMS."""
    from ibl import datasets
    from ibl.utils.data import get_transformer_test
    from oracle import ibl_oracle as O
    base = tmp_path_factory.mktemp("tokyo_eval")
    src = str(base / "src")
    datasets.write_synthetic_pitts_tree(os.path.join(src, "pitts"), scale="30k")
    datasets.write_synthetic_tokyo_tree(os.path.join(src, "tokyo"), n_places=(12, 9, 24), seed=2)
    ckpt = str(base / "model_best.pth.tar")
    sd = _checkpoint(ckpt)
    work = str(base / "oracle")
    shutil.copytree(src, work)
    pitts = datasets.create("pitts", os.path.join(work, "pitts"), scale="30k", verbose=False)
    tokyo = datasets.create("tokyo", os.path.join(work, "tokyo"), verbose=False)
    train = sorted(list(set(pitts.q_train) | set(pitts.db_train)))
    U, lams, mu, _ = O.pca_train(_oracle_feats(pitts, train, get_transformer_test(H, W), sd), n_components=FEATURES)
    pca = O.pca_load(U, lams, mu, n_components=FEATURES)
    q = _oracle_feats(tokyo, tokyo.q_test, get_transformer_test(H, W, tokyo=True), sd, pca)
    db = _oracle_feats(tokyo, tokyo.db_test, get_transformer_test(H, W), sd, pca)
    want = O.evaluate_all(O.pairwise_distance(q, db).numpy(), tokyo.test_pos, [g[1] for g in tokyo.db_test], nms=True)
    assert 0 < want[0] <= 1
    return dict(base=str(base), src=src, ckpt=ckpt, want=want, n_q=len(tokyo.q_test))


@pytest.mark.parametrize("nproc", [1, pytest.param(2, marks=pytest.mark.skipif(not TWO_GPUS, reason="needs two GPUs"))])
def test_reference_examples_test_py_on_tokyo_matches_oracle(eval_setup, nproc):
    data = open(TEST_PY, "rb").read()
    assert hashlib.sha256(data).hexdigest() == TEST_PY_SHA256
    run = os.path.join(eval_setup["base"], "run%d" % nproc)
    data_dir, logs = os.path.join(run, "data"), os.path.join(run, "logs")
    shutil.copytree(eval_setup["src"], data_dir)
    os.makedirs(logs)
    ckpt = os.path.join(logs, "model_best.pth.tar")
    shutil.copy(eval_setup["ckpt"], ckpt)
    script = os.path.join(run, "test.py")
    with open(script, "wb") as f:
        f.write(data)
    env = dict(os.environ, IBL_VGG16_RANDOM_INIT_OK="1",
               PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests", "fixtures", "stubs"),
                                           os.environ.get("PYTHONPATH", "")]))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(29780 + nproc),
           script, "--launcher", "pytorch", "-d", "tokyo", "--data-dir", data_dir, "--resume", ckpt,
           "--vlad", "--reduction", "--features", str(FEATURES), "--height", str(H), "--width", str(W),
           "--test-batch-size", "8", "-j", "2"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=run, env=env)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    assert all(os.path.isfile(os.path.join(data_dir, "tokyo", n)) for n in ("meta.json", "splits.json"))
    log = open(os.path.join(logs, "log_test_tokyo.txt")).read()
    assert "calculating PCA parameters" in out.stdout + log
    got = [float(v) for v in re.findall(r"top-(?:1|5|10)\s+([0-9.]+)%", log)[-3:]]
    assert len(got) == 3, log[-2000:]
    assert np.allclose(got, np.round(100 * eval_setup["want"], 1), atol=0.051), (got, eval_setup["want"])


# ---- examples/cluster.py + examples/netvlad_img.py -d tokyo ---------------------------------------------------------
def _env(**extra):
    env = dict(os.environ, IBL_VGG16_RANDOM_INIT_OK="1",
               PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests", "fixtures", "stubs_h5npz"),
                                           os.environ.get("PYTHONPATH", "")]))
    env.update(extra)
    return env


@pytest.fixture(scope="module")
def recipe(tmp_path_factory):
    """A synthetic Tokyo tree with 528 Time Machine training images, the seeded base weights, and cluster.py's
    centroid file for `-d tokyo` (cluster.py arranges the tree on its first dataset creation)."""
    base = str(tmp_path_factory.mktemp("tokyo_recipe"))
    os.makedirs(os.path.join(base, "examples"))
    for name, sha in SCRIPTS.items():
        data = open(os.path.join(GOLDEN, f"reference_examples_{name}.py.txt"), "rb").read()
        assert hashlib.sha256(data).hexdigest() == sha, name
        with open(os.path.join(base, "examples", name + ".py"), "wb") as f:
            f.write(data)
    from ibl import datasets
    data_dir = os.path.join(base, "data")
    datasets.write_synthetic_tokyo_tree(os.path.join(data_dir, "tokyo"), n_places=(TM_TRAIN_PLACES, 12, 12),
                                        size=(RH, RW), seed=3)
    logs = os.path.join(base, "logs")
    os.makedirs(logs)
    vgg = {k[len("base."):]: v for k, v in synth.make_vgg_weights(3, 0.0).items()}
    torch.save(vgg, os.path.join(logs, "vd16_offtheshelf_conv5_3_max.pth"))
    cmd = [sys.executable, os.path.join(base, "examples", "cluster.py"), "-d", "tokyo", "--data-dir", data_dir,
           "--logs-dir", logs, "-b", "64", "-j", "2", "--height", str(RH), "--width", str(RW), "--seed", "43"]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=base, env=_env(CUDA_VISIBLE_DEVICES="0"))
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    with np.load(os.path.join(logs, "vgg16_tokyo_64_desc_cen.hdf5")) as z:
        desc, cent = z["descriptors"].copy(), z["centroids"].copy()
    ds = datasets.create("tokyo", os.path.join(data_dir, "tokyo"), verbose=False)
    assert ds.q_val and ds.db_val and len(set(ds.q_train) | set(ds.db_train)) >= 500
    assert {it[0] for it in ds.q_train} == {it[0] for it in ds.db_train}          # q_train == db_train
    return dict(base=base, data_dir=data_dir, logs=logs, ds=ds, vgg=vgg, desc=desc, cent=cent)


def test_netvlad_img_py_trains_one_epoch_on_tokyo_time_machine(recipe):
    base, logs = recipe["base"], os.path.join(recipe["base"], "run")
    nproc = 2 if TWO_GPUS else 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", "29785",
           os.path.join(base, "examples", "netvlad_img.py"), "--launcher", "pytorch", "-d", "tokyo",
           "--data-dir", recipe["data_dir"], "--init-dir", recipe["logs"], "--logs-dir", logs,
           "--vlad", "--loss-type", "triplet", "--tuple-size", "1", "--neg-num", "3", "--epochs", "1", "--iters", "2",
           "--height", str(RH), "--width", str(RW), "--test-batch-size", "16", "-j", "4",
           "--features", str(FEATURES), "--print-freq", "1"]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, cwd=base, env=_env())
    log_path = os.path.join(logs, "log.txt")
    log = open(log_path).read() if os.path.isfile(log_path) else ""
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:] + log[-2000:]
    losses = [float(v) for v in re.findall(r"Epoch: \[0-0\]\[[12]/2\].*Loss ([0-9.]+)", log)]
    assert len(losses) == 2 and all(np.isfinite(losses)), log[-3000:]
    assert re.search(r"Finished epoch\s+0 recall@1:\s*[0-9.]+%\s+recall@5:\s*[0-9.]+%", log), log[-3000:]
    assert os.path.isfile(os.path.join(logs, "checkpoint0.pth.tar"))
    tail = log[log.rindex("Testing on Pitts30k-test"):]                # the script's label; the split is Tokyo 24/7
    assert len(re.findall(r"top-(?:1|5|10)\s+([0-9.]+)%", tail)) >= 3, tail[-2000:]


def test_first_training_step_on_a_time_machine_tuple_matches_oracle(recipe):
    """netvlad_img.py's first step: the model it starts from (the base weights, NetVLAD initialised from cluster.py's
    centroids), the gallery ranking update_sampler computes, then the first tuple DistributedRandomTupleSampler deals
    after `random.seed(43)`.  The engine's triplet loss on that tuple equals the CPU oracle's."""
    from torch.utils.data import DataLoader
    from ibl import models
    from ibl.evaluators import extract_features, pairwise_distance
    from ibl.trainers import Trainer
    from ibl.utils.data import get_transformer_test, get_transformer_train
    from ibl.utils.data.preprocessor import Preprocessor
    from ibl.utils.data.sampler import DistributedRandomTupleSampler
    from oracle import ibl_oracle as O
    ds = recipe["ds"]
    base = models.create("vgg16", pretrained=False)
    base.base.load_state_dict(recipe["vgg"])
    pool = models.create("netvlad", dim=512)
    pool.clsts, pool.traindescs = recipe["cent"], recipe["desc"]
    pool._init_params()
    model = models.create("embednet", base, pool)
    for layer in list(model.base_model.base.children())[:24]:
        for p in layer.parameters():
            p.requires_grad = False
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    model = model.cuda()

    train = sorted(list(set(ds.q_train) | set(ds.db_train)))
    loader = DataLoader(Preprocessor(train, root=ds.images_dir, transform=get_transformer_test(RH, RW)),
                        batch_size=16, num_workers=2, shuffle=False)
    feats = extract_features(model, loader, train, print_freq=1000)
    distmat, _, _ = pairwise_distance(feats, ds.q_train, ds.db_train)
    sampler = DistributedRandomTupleSampler(ds.q_train, ds.db_train, ds.train_pos, ds.train_neg, neg_num=3,
                                            neg_pool=1000, num_replicas=1, rank=0)
    g = torch.Generator()
    g.manual_seed(43)
    sampler.sort_gallery(distmat, torch.randperm(len(ds.q_train), generator=g).long().tolist())
    random.seed(43)
    tup = next(iter(sampler))
    items = ds.q_train + ds.db_train
    assert items[tup[1]][1] != items[tup[0]][1]                  # the positive is another time stamp or place

    pre = Preprocessor(items, root=ds.images_dir, transform=get_transformer_train(RH, RW))
    torch.manual_seed(0)                                         # the colour-jitter draws
    x = torch.stack([pre[i][0] for i in tup])[None]               # [1, 2 + neg_num, 3, RH, RW]
    loss = Trainer(model.train(), margin=MARGIN, gpu=0)._forward(x.cuda(), True, "triplet")
    with torch.no_grad():
        _, v = O.embednet_forward(x[0], sd)
    want = F.triplet_margin_loss(v[:1].expand(3, -1), v[1:2].expand(3, -1), v[2:], margin=MARGIN, p=2).item()
    assert np.isfinite(want) and abs(loss.item() - want) < 2e-4 * max(1.0, abs(want)), (loss.item(), want)


# ---- device decode of Tokyo 24/7 queries ----------------------------------------------------------------------------
def test_tokyo_queries_decode_on_the_device_bit_identical(eval_setup, monkeypatch, tmp_path):
    from torch.utils.data import DataLoader
    from ibl import datasets
    from ibl.evaluators import extract_features
    from ibl.utils.data import get_transformer_test
    from ibl.utils.data.preprocessor import Preprocessor
    from openibl_b200.utils.data import gpu_jpeg
    root = str(tmp_path / "tokyo")
    shutil.copytree(os.path.join(eval_setup["src"], "tokyo"), root)
    ds = datasets.create("tokyo", root, verbose=False)
    sizes = {open_size(os.path.join(ds.images_dir, it[0])) for it in ds.q_test}
    assert any(w > h for w, h in sizes) and any(h > w for w, h in sizes), sizes

    from ibl import models
    torch.manual_seed(3)
    base = models.create("vgg16", pretrained=False)
    pool = models.create("netvlad", dim=base.feature_dim)
    p = synth.make_netvlad_params(seed=3, sharp=True)
    pool.centroids.data.copy_(p["centroids"])
    pool.conv.weight.data.copy_(p["conv_weight"])
    model = models.create("embednet", base, pool).cuda()

    def loader(device_decode):
        tf = get_transformer_test(H, W, tokyo=True, device_decode=device_decode)
        return DataLoader(Preprocessor(ds.q_test, root=ds.images_dir, transform=tf), batch_size=1, num_workers=0,
                          shuffle=False)

    host = extract_features(model, loader(False), ds.q_test, print_freq=1000)

    def refuse(data):
        raise AssertionError("a Tokyo query reached the host decoder")
    monkeypatch.setattr(gpu_jpeg, "_host_decode", refuse)
    dev = extract_features(model, loader(True), ds.q_test, print_freq=1000)
    assert list(host) == list(dev)
    for k in host:
        assert torch.equal(host[k], dev[k]), k
    from PIL import Image
    host_tf = get_transformer_test(H, W, tokyo=True)
    shapes = set()
    for it in ds.q_test:
        path = os.path.join(ds.images_dir, it[0])
        want = host_tf(Image.open(path).convert("RGB"))
        got = gpu_jpeg.decode_to_tensor([open(path, "rb").read()], H, W, tokyo=True).cpu()[0]
        assert torch.equal(got, want), it[0]
        shapes.add(tuple(want.shape))
    assert len(shapes) >= 3, shapes                           # Resize(max(H, W)) gives several output sizes


def open_size(path):
    from PIL import Image
    with Image.open(path) as im:
        return im.size

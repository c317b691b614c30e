"""NetVLAD / SARE training on the engine (`ibl.trainers.Trainer`, examples/netvlad_img.py):

* one training step per golden case against the UNMODIFIED reference run on CPU (tests/golden/trainer_step.npz,
  oracle/gen_golden_trainer.py): triplet / sare_ind / sare_joint on `EmbedNet`'s VLAD, and triplet on the bare
  `VGG`'s max-pooled feature (vlad=False);
* one `Trainer.train` step under DistributedDataParallel, launched with torch.distributed.run;
* the reference's training recipe, run as the byte-identical scripts (vendored as test data next to the goldens):
  examples/cluster.py writes the NetVLAD centroid file, then examples/netvlad_img.py trains, validates, saves, fits
  the PCA and tests, on a Pittsburgh-shaped synthetic tree; its final recalls must equal the CPU oracle's;
* cluster.py under nn.DataParallel over two GPUs (when two are present) against a one-GPU run."""
import hashlib
import os
import re
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT, load_golden, rel_l2
from openibl_b200 import synth

pytestmark = pytest.mark.gpu

B, NEG, H, W, SEED = 2, 3, 64, 96, 13          # oracle/gen_golden_trainer.py
CASES = [("triplet", True), ("sare_ind", True), ("sare_joint", True), ("triplet", False)]
TWO_GPUS = torch.cuda.is_available() and torch.cuda.device_count() >= 2


def _freeze_below_conv5(trunk):
    for layer in list(trunk.base.children())[:24]:
        for p in layer.parameters():
            p.requires_grad = False


def _build(vlad):
    from ibl import models
    base = models.create("vgg16", pretrained=False)
    if vlad:
        m = models.create("embednet", base, models.create("netvlad", dim=512))
        m.load_state_dict(synth.make_state_dict(seed=SEED, sharp=True, with_pca=False, bias_scale=0.02))
        trunk = m.base_model
    else:
        m = base
        m.load_state_dict(synth.make_vgg_weights(SEED, 0.02))
        trunk = m
    _freeze_below_conv5(trunk)
    return m.cuda().train(), trunk


@pytest.mark.parametrize("loss_type,vlad", CASES, ids=[f"{l}-{'vlad' if v else 'pool'}" for l, v in CASES])
def test_trainer_step_losses_and_gradients_vs_reference_golden(loss_type, vlad):
    """Loss within 2e-4 relative of the unmodified reference on CPU; NetVLAD gradients within 3e-3 relative L2; conv5
    gradients within 2e-2 and cosine > 0.9998 -- the tolerances of the SFRS step test, for the same reason: an
    activation whose pre-activation is within fp32 noise of zero takes a different side of a conv5 ReLU in the two
    implementations, and each flip switches a gradient path."""
    from ibl.trainers import Trainer
    g = load_golden("trainer_step")
    name = f"{loss_type}_{'vlad' if vlad else 'pool'}"
    easy, _ = synth.make_sfrs_tuples(seed=41, tuples=B, neg_num=NEG, n_diff=1, height=H, width=W)
    model, trunk = _build(vlad)
    loss = Trainer(model, margin=0.1 ** 0.5, gpu=0)._forward(easy.cuda(), vlad, loss_type)
    want = float(g[f"{name}_loss"])
    assert abs(loss.item() - want) < 2e-4 * max(1.0, abs(want)), (loss.item(), want)
    loss.backward()
    base = trunk.base
    assert base[21].weight.grad is None and base[21].bias.grad is None          # frozen below conv5
    for slot in (24, 26, 28):
        gw = base[slot].weight.grad.cpu()
        sub, ref = gw[::16, ::8].double().flatten(), torch.from_numpy(g[f"{name}_w{slot}"]).double().flatten()
        assert rel_l2(sub, ref) < 2e-2, (slot, rel_l2(sub, ref))
        assert float(sub @ ref / (sub.norm() * ref.norm())) > 0.9998, slot
        wnorm = float(g[f"{name}_w{slot}_norm"])
        assert abs(float(gw.double().norm()) - wnorm) < 1e-2 * wnorm
        # conv5_3 has no ReLU, and max-pooling commutes with its bias: with the max-pooled descriptor the triplet loss
        # is invariant to that bias, whose gradient is zero up to rounding in both implementations (a norm ~1e-7 of
        # the weight gradient's), so the relative test gets an absolute floor at that scale
        gb, want_b = base[slot].bias.grad.cpu().double(), torch.from_numpy(g[f"{name}_b{slot}"]).double()
        assert float((gb - want_b).norm()) < 2e-2 * float(want_b.norm()) + 1e-5 * wnorm, (slot, rel_l2(gb, want_b))
    if vlad:
        assert rel_l2(model.net_vlad.centroids.grad.cpu()[:, ::4], g[f"{name}_centroids"]) < 3e-3
        assert rel_l2(model.net_vlad.conv.weight.grad.cpu()[:, ::4, 0, 0], g[f"{name}_conv_w"]) < 3e-3


def test_engine_get_from_concurrent_threads_returns_one_engine_per_device():
    """nn.DataParallel calls the replicas from one thread per device: concurrent first calls must agree."""
    from openibl_b200 import engine as E
    got, errors = [], []

    def worker(dev):
        try:
            got.append((dev, E.Engine.get(dev)))
        except Exception as exc:     # pragma: no cover
            errors.append(exc)

    devs = list(range(torch.cuda.device_count())) * 4
    threads = [threading.Thread(target=worker, args=(d,)) for d in devs]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors
    for dev, eng in got:
        assert eng is E._engines[dev] and eng.device == dev


# ---- DistributedDataParallel step -------------------------------------------------------------------------------
DDP_WORKER = r'''
import json, os, sys
sys.path.insert(0, {root!r})
import torch, torch.distributed as dist
from ibl import models
from ibl.trainers import Trainer
from openibl_b200 import synth

rank = int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl")
m = models.create("embednet", models.create("vgg16", pretrained=False), models.create("netvlad", dim=512))
m.load_state_dict(synth.make_state_dict(seed=13, sharp=True, with_pca=False, bias_scale=0.02))
for layer in list(m.base_model.base.children())[:24]:
    for p in layer.parameters():
        p.requires_grad = False
m.cuda(rank)
before = {{k: v.detach().clone() for k, v in m.state_dict().items()}}
model = torch.nn.parallel.DistributedDataParallel(m, device_ids=[rank], output_device=rank, find_unused_parameters=True)
opt = torch.optim.SGD(filter(lambda p: p.requires_grad, model.parameters()), lr=0.01, momentum=0.9, weight_decay=0.001)


class Loader:                     # IterLoader's interface; each rank gets different tuples, as the sampler deals them
    def new_epoch(self):
        pass

    def next(self):
        easy, _ = synth.make_sfrs_tuples(seed=50 + rank, tuples=2, neg_num=3, n_diff=1, height=64, width=96)
        return [(easy[:, j], ["f"] * 2, torch.zeros(2), torch.zeros(2), torch.zeros(2)) for j in range(easy.shape[1])]


Trainer(model, margin=0.1 ** 0.5, gpu=rank).train(0, 0, Loader(), opt, train_iters=1, print_freq=1, vlad=True,
                                                   loss_type={loss!r})
equal, changed, frozen = True, [], []
for k, v in m.state_dict().items():
    parts = [torch.empty_like(v) for _ in range(dist.get_world_size())]
    dist.all_gather(parts, v.contiguous())
    equal = equal and all(torch.equal(p, parts[0]) for p in parts)
    (changed if not torch.equal(v, before[k]) else frozen).append(k)
if rank == 0:
    json.dump({{"equal": equal, "changed": changed, "unchanged": frozen, "world": dist.get_world_size()}},
              open({out!r}, "w"))
dist.barrier()
dist.destroy_process_group()
'''


@pytest.mark.parametrize("loss_type", ["triplet", "sare_ind"])
def test_trainer_step_under_ddp_keeps_ranks_in_sync(tmp_path, loss_type):
    """One `Trainer.train` step (tuple_size 2, DDP with find_unused_parameters=True as netvlad_img.py:107-109 sets it):
    afterwards every parameter is identical on all ranks, conv5 and NetVLAD moved, conv1-conv4 did not."""
    import json
    out = str(tmp_path / "ddp.json")
    script = tmp_path / "ddp_step.py"
    script.write_text(DDP_WORKER.format(root=ROOT, out=out, loss=loss_type))
    nproc = 2 if TWO_GPUS else 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(29751 + ["triplet", "sare_ind"].index(loss_type)), str(script)]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=str(tmp_path))
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert re.search(r"Epoch: \[0-0\]\[1/1\].*Loss [0-9.]+", res.stdout), res.stdout[-2000:]
    r = json.load(open(out))
    assert r["world"] == nproc and r["equal"]
    trained = {f"base_model.base.{s}.{t}" for s in (24, 26, 28) for t in ("weight", "bias")}
    trained |= {"net_vlad.centroids", "net_vlad.conv.weight"}
    assert set(r["changed"]) == trained, r["changed"]


# ---- the reference's training recipe, unmodified ---------------------------------------------------------------
SCRIPTS = {"cluster": "785c1fcf8219c58fdbbb4be5cc7df7013174162b18fe3db7853256f1b0a68452",
           "netvlad_img": "9f2c21800b4cadc563d4e3072dc5b74c193f3133070574391d2429c7e9adbbd5"}
RH, RW = 160, 256                 # conv5 map 10 x 16 = 160 locations >= the 100 cluster.py samples per image
N_TRAIN_PLACES = 208              # 2 views per place + a query for every second place: 520 >= the 500 cluster.py samples
FEATURES = 32


def _install_scripts(base):
    os.makedirs(os.path.join(base, "examples"), exist_ok=True)
    for name, sha in SCRIPTS.items():
        data = open(os.path.join(GOLDEN, f"reference_examples_{name}.py.txt"), "rb").read()
        assert hashlib.sha256(data).hexdigest() == sha, name
        with open(os.path.join(base, "examples", name + ".py"), "wb") as f:
            f.write(data)


def _env(**extra):
    # models.create('vgg16') defaults to pretrained=True (a download); the scripts then load the seeded base weights
    # from logs/vd16_offtheshelf_conv5_3_max.pth.  The npz-backed h5py stand-in serves their h5py.File calls, also in
    # the DataLoader workers.
    env = dict(os.environ, IBL_VGG16_RANDOM_INIT_OK="1",
               PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests", "fixtures", "stubs_h5npz"),
                                           os.environ.get("PYTHONPATH", "")]))
    env.update(extra)
    return env


def _run_cluster(base, data_dir, logs, env):
    cmd = [sys.executable, os.path.join(base, "examples", "cluster.py"), "-d", "pitts", "--data-dir", data_dir,
           "--logs-dir", logs, "-b", "64", "-j", "2", "--height", str(RH), "--width", str(RW), "--seed", "43"]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=base, env=env)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    with np.load(os.path.join(logs, "vgg16_pitts_64_desc_cen.hdf5")) as z:
        return z["descriptors"].copy(), z["centroids"].copy()


@pytest.fixture(scope="module")
def recipe(tmp_path_factory):
    """A synthetic Pittsburgh tree, the seeded base weights and cluster.py's centroid file (one GPU visible)."""
    from ibl import datasets
    base = str(tmp_path_factory.mktemp("recipe"))
    _install_scripts(base)
    data_dir = os.path.join(base, "data")
    datasets.write_synthetic_pitts_tree(os.path.join(data_dir, "pitts"), scale="30k",
                                        n_places=(N_TRAIN_PLACES, 24, 16), size=(RH, RW))
    ds = datasets.create("pitts", os.path.join(data_dir, "pitts"), scale="30k", verbose=False)
    assert len(set(ds.q_train) | set(ds.db_train)) >= 500
    assert all(len(p) > 0 for p in ds.train_pos), "every training query needs a positive"
    logs = os.path.join(base, "logs")
    os.makedirs(logs)
    vgg = {k[len("base."):]: v for k, v in synth.make_vgg_weights(3, 0.0).items()}
    torch.save(vgg, os.path.join(logs, "vd16_offtheshelf_conv5_3_max.pth"))
    desc, cent = _run_cluster(base, data_dir, logs, _env(CUDA_VISIBLE_DEVICES="0"))
    return dict(base=base, data_dir=data_dir, logs=logs, ds=ds, vgg=vgg, desc=desc, cent=cent)


def test_cluster_py_writes_unit_norm_descriptors_and_centroids(recipe):
    desc, cent = recipe["desc"], recipe["cent"]
    assert desc.shape == (50000, 512) and cent.shape == (64, 512)
    assert np.allclose(np.linalg.norm(desc, axis=1), 1.0, atol=1e-5)
    assert np.isfinite(cent).all()


def _initial_netvlad(recipe):
    from ibl import models
    nv = models.create("netvlad", dim=512)
    nv.clsts, nv.traindescs = recipe["cent"], recipe["desc"]
    nv._init_params()
    return nv.centroids.detach().clone(), nv.conv.weight.detach().clone()


def _oracle_recalls(recipe, sd, pca_path):
    from ibl.utils.data import get_transformer_test
    from ibl.utils.data.preprocessor import Preprocessor
    from oracle import ibl_oracle as O
    ds = recipe["ds"]
    tf = get_transformer_test(RH, RW)

    def feats(items):
        pre = Preprocessor(items, root=ds.images_dir, transform=tf)
        x = torch.stack([pre[i][0] for i in range(len(items))])
        with torch.no_grad():
            return O.extract_descriptor(x, sd, vlad=True)

    with np.load(pca_path) as p:            # the PCA file the run wrote, through the npz-backed h5py stand-in
        w, b = O.pca_load(p["U"], p["lams"], p["mu"], n_components=FEATURES)
    q = O.pca_whiten(feats(ds.q_test), w, b)
    db = O.pca_whiten(feats(ds.db_test), w, b)
    return O.evaluate_all(O.pairwise_distance(q, db).numpy(), ds.test_pos, [g[1] for g in ds.db_test])


@pytest.mark.parametrize("loss_type", ["triplet", "sare_ind"])
def test_netvlad_img_py_trains_unmodified_and_matches_oracle(recipe, loss_type):
    base, logs = recipe["base"], os.path.join(recipe["base"], "run_" + loss_type)
    nproc = 2 if TWO_GPUS else 1
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(29761 + ["triplet", "sare_ind"].index(loss_type)),
           os.path.join(base, "examples", "netvlad_img.py"), "--launcher", "pytorch", "-d", "pitts", "--scale", "30k",
           "--data-dir", recipe["data_dir"], "--init-dir", recipe["logs"], "--logs-dir", logs,
           "--vlad", "--loss-type", loss_type, "--tuple-size", "1", "--neg-num", "3", "--epochs", "1", "--iters", "2",
           "--cache-size", "52", "--height", str(RH), "--width", str(RW), "--test-batch-size", "16", "-j", "4",
           "--features", str(FEATURES), "--print-freq", "1"]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, cwd=base, env=_env())
    log_path = os.path.join(logs, "log.txt")
    log = open(log_path).read() if os.path.isfile(log_path) else ""
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:] + log[-2000:]
    # two cache subsets (104 training queries, --cache-size 52), two iterations each
    assert len(re.findall(r"Epoch: \[0-[01]\]\[[12]/2\].*Loss [0-9.]+", log)) == 4, log[-3000:]
    # model_best.pth.tar exists only if validation Recall@5 beat the initial 0 (netvlad_img.py:197)
    m = re.search(r"Finished epoch\s+0 recall@1:\s*([0-9.]+)%\s+recall@5:\s*([0-9.]+)%", log)
    assert m and float(m.group(2)) > 0, log[-3000:]
    assert os.path.isfile(os.path.join(logs, "checkpoint0.pth.tar"))
    best = os.path.join(logs, "model_best.pth.tar")
    assert os.path.isfile(best)
    sd = {k[len("module."):]: v for k, v in torch.load(best, map_location="cpu", weights_only=False)["state_dict"].items()}
    for slot in synth.VGG16_CONV_SLOTS:
        w0, w1 = recipe["vgg"][f"{slot}.weight"], sd[f"base_model.base.{slot}.weight"]
        if slot < 24:
            assert torch.equal(w0, w1), slot                  # conv1-conv4: frozen
        else:
            assert not torch.equal(w0, w1), slot              # conv5: trained
    c0, w0 = _initial_netvlad(recipe)
    assert not torch.equal(sd["net_vlad.centroids"], c0) and not torch.equal(sd["net_vlad.conv.weight"], w0)
    # the final "Testing on Pitts30k-test" recalls equal the CPU oracle's for model_best and the run's PCA file
    tail = log[log.rindex("Testing on Pitts30k-test"):]
    got = [float(v) for v in re.findall(r"top-(?:1|5|10)\s+([0-9.]+)%", tail)[-3:]]
    assert len(got) == 3, tail[-2000:]
    want = _oracle_recalls(recipe, sd, os.path.join(logs, "pca_params_model_best.h5"))
    assert np.allclose(got, np.round(100 * want, 1), atol=0.051), (got, want)


@pytest.mark.skipif(not TWO_GPUS, reason="needs two GPUs")
def test_cluster_py_under_data_parallel_on_two_gpus_matches_one_gpu(recipe, tmp_path):
    """nn.DataParallel splits each batch over both GPUs (one engine per device, each in its own thread, on freshly
    replicated parameters every forward); the descriptors equal the one-GPU run with the same seed."""
    logs = str(tmp_path / "logs2")
    os.makedirs(logs)
    desc, _ = _run_cluster(recipe["base"], recipe["data_dir"], logs, _env(CUDA_VISIBLE_DEVICES="0,1"))
    assert desc.shape == recipe["desc"].shape
    assert np.allclose(desc, recipe["desc"], rtol=0, atol=1e-5), np.abs(desc - recipe["desc"]).max()

"""The reference's third training step, examples/netvlad_img_sfrs.py (SFRS), run as the byte-identical script (vendored
next to the goldens, sha256-pinned) on the synthetic Pittsburgh tree and centroid file of test_gpu_trainer.py's
recipe.  Two generations of one epoch: generation 1 refreshes the sampler with k-reciprocal re-ranking of host
distance matrices (re_ranking's device route) and trains with the soft loss; the final test recalls must equal the
CPU oracle's for the run's best model and PCA file."""
import hashlib
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from openibl_b200 import synth
from test_gpu_trainer import FEATURES, RH, RW, TWO_GPUS, _env, _initial_netvlad, _oracle_recalls, recipe  # noqa: F401

pytestmark = pytest.mark.gpu

SFRS_SHA256 = "3dcab77228ce759f6789b7b06315fee66ed20f8b2178e4b7449f023e2c6c7bd3"


def _install_sfrs(base):
    data = open(os.path.join(GOLDEN, "reference_examples_netvlad_img_sfrs.py.txt"), "rb").read()
    assert hashlib.sha256(data).hexdigest() == SFRS_SHA256
    path = os.path.join(base, "examples", "netvlad_img_sfrs.py")
    with open(path, "wb") as f:
        f.write(data)
    return path


def test_netvlad_img_sfrs_py_trains_two_generations_and_matches_oracle(recipe):  # noqa: F811
    base, logs = recipe["base"], os.path.join(recipe["base"], "run_sfrs")
    script = _install_sfrs(base)
    nproc = 2 if TWO_GPUS else 1
    # every training query has two positives (the two views of its place): --pos-num / --pos-pool 2
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", "29781", script, "--launcher", "pytorch", "-d", "pitts",
           "--scale", "30k", "--data-dir", recipe["data_dir"], "--init-dir", recipe["logs"], "--logs-dir", logs,
           "--tuple-size", "1", "--neg-num", "3", "--pos-num", "2", "--pos-pool", "2", "--generations", "2",
           "--epochs", "1", "--iters", "2", "--cache-size", "52", "--height", str(RH), "--width", str(RW),
           "--test-batch-size", "16", "-j", "4", "--features", str(FEATURES), "--print-freq", "1"]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1800, cwd=base, env=_env())
    log_path = os.path.join(logs, "log.txt")
    log = open(log_path).read() if os.path.isfile(log_path) else ""
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:] + log[-2000:]
    for name in ("checkpoint0_0.pth.tar", "checkpoint1_0.pth.tar", "model_best.pth.tar", "pca_params_model_best.h5"):
        assert os.path.isfile(os.path.join(logs, name)), name
    g0 = re.search(r"Finished generation\s+0 epoch\s+0", log)
    assert g0 and re.search(r"Finished generation\s+1 epoch\s+0", log), log[-3000:]
    # generation 1: two cache subsets (104 training queries, --cache-size 52), two iterations each, with the soft loss
    gen1 = log[g0.end():]
    soft = re.findall(r"Epoch: \[0-[01]\]\[[12]/2\].*Loss_soft ([0-9.]+)", gen1)
    assert len(soft) == 4, gen1[-3000:]
    sd = {k[len("module."):]: v
          for k, v in torch.load(os.path.join(logs, "model_best.pth.tar"), map_location="cpu",
                                 weights_only=False)["state_dict"].items()}
    for slot in synth.VGG16_CONV_SLOTS:
        w0, w1 = recipe["vgg"][f"{slot}.weight"], sd[f"base_model.base.{slot}.weight"]
        if slot < 24:
            assert torch.equal(w0, w1), slot                  # conv1-conv4: frozen
        else:
            assert not torch.equal(w0, w1), slot              # conv5: trained
    c0, w0 = _initial_netvlad(recipe)
    assert not torch.equal(sd["net_vlad.centroids"], c0) and not torch.equal(sd["net_vlad.conv.weight"], w0)
    tail = log[log.rindex("Testing on Pitts30k-test"):]
    got = [float(v) for v in re.findall(r"top-(?:1|5|10)\s+([0-9.]+)%", tail)[-3:]]
    assert len(got) == 3, tail[-2000:]
    want = _oracle_recalls(recipe, sd, os.path.join(logs, "pca_params_model_best.h5"))
    assert np.allclose(got, np.round(100 * want, 1), atol=0.051), (got, want)

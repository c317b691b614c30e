"""NetVLAD / SARE training on the host side: `Trainer._get_loss` (ibl/trainers.py:82-162) against the unmodified
reference trainer (tests/golden/trainer_step.npz, oracle/gen_golden_trainer.py), the unknown-loss error, and the
imports of the reference's training recipe (examples/cluster.py, netvlad_img.py, netvlad_img_sfrs.py)."""
import ast
import hashlib
import importlib
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT, load_golden

LOSSES = ("triplet", "sare_ind", "sare_joint")
SHAPES = ((1, 3), (2, 5), (4, 12), (3, 4))      # (B, N) of the golden loss cases


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("loss_type", LOSSES)
def test_trainer_loss_and_gradient_match_reference_golden(loss_type, shape):
    """The Euclidean triplet / SARE losses and their gradient w.r.t. the descriptors, on random descriptors, within
    fp32 noise of the reference (the same formulas; only the order of a few reductions may differ)."""
    from ibl.trainers import Trainer
    g = load_golden("trainer_step")
    b, n = shape
    key = f"u{b}x{n}"
    tr = Trainer(None, margin=0.1 ** 0.5, gpu=None)
    o = torch.from_numpy(g[f"{key}_outputs"]).clone().requires_grad_(True)
    loss = tr._get_loss(o, loss_type, b, n)
    loss.backward()
    want = float(g[f"{key}_{loss_type}_loss"])
    assert abs(loss.item() - want) < 2e-6 * max(1.0, abs(want)), (loss.item(), want)
    assert np.allclose(o.grad.numpy(), g[f"{key}_{loss_type}_grad"], rtol=1e-5, atol=1e-7)


def test_trainer_unknown_loss_raises_value_error():
    from ibl.trainers import Trainer
    with pytest.raises(ValueError, match="Unknown loss function"):
        Trainer(None)._get_loss(torch.randn(6, 8), "contrastive", 2, 3)


def test_trainer_constructor_defaults():
    """Same defaults as the reference (trainers.py:17)."""
    from ibl.trainers import Trainer
    tr = Trainer("model")
    assert (tr.model, tr.margin, tr.gpu, tr.temp) == ("model", 0.3, None, 0.07)


# every `from ibl... import ...` of the reference's training recipe (examples/cluster.py:17-24,
# netvlad_img.py:20-30, netvlad_img_sfrs.py:19-30)
RECIPE_IMPORTS = {
    "ibl": ["datasets", "models"],
    "ibl.trainers": ["Trainer", "SFRSTrainer"],
    "ibl.evaluators": ["Evaluator", "extract_features", "pairwise_distance"],
    "ibl.utils.data": ["IterLoader", "get_transformer_train", "get_transformer_test"],
    "ibl.utils.data.sampler": ["DistributedRandomTupleSampler", "DistributedRandomDiffTupleSampler",
                               "DistributedSliceSampler", "SubsetRandomSampler"],
    "ibl.utils.data.preprocessor": ["Preprocessor"],
    "ibl.utils.logging": ["Logger"],
    "ibl.pca": ["PCA"],
    "ibl.utils.serialization": ["load_checkpoint", "save_checkpoint", "copy_state_dict"],
    "ibl.utils.dist_utils": ["init_dist", "synchronize", "convert_sync_bn"],
    "ibl.utils.rerank": ["re_ranking"],
}


def test_every_name_the_training_recipe_imports_resolves():
    for mod, names in RECIPE_IMPORTS.items():
        m = importlib.import_module(mod)
        for name in names:
            assert hasattr(m, name), f"{mod}.{name}"


@pytest.mark.parametrize("script", ["cluster", "netvlad_img"])
def test_vendored_recipe_scripts_import_only_resolvable_ibl_names(script):
    """The vendored copies of examples/cluster.py and netvlad_img.py (the GPU drop-in test runs them): every
    `from ibl... import name` they contain resolves, and the list above covers it."""
    path = os.path.join(GOLDEN, f"reference_examples_{script}.py.txt")
    tree = ast.parse(open(path, "rb").read().decode())
    found = [(n.module, a.name) for n in ast.walk(tree) if isinstance(n, ast.ImportFrom) and n.module
             and n.module.split(".")[0] == "ibl" for a in n.names]
    assert found
    for mod, name in found:
        assert name in RECIPE_IMPORTS[mod], (mod, name)
        assert hasattr(importlib.import_module(mod), name), (mod, name)


def test_sampler_module_reexports_torch_samplers():
    import torch.utils.data as tud
    from ibl.utils.data import sampler
    for name in ("SequentialSampler", "RandomSampler", "SubsetRandomSampler", "WeightedRandomSampler", "BatchSampler"):
        assert getattr(sampler, name) is getattr(tud, name), name


def test_npz_h5py_stand_in_round_trip(tmp_path):
    """The npz-backed `h5py` stand-in the drop-in recipe test runs the scripts with: the calls cluster.py,
    netvlad_img.py and the PCA store make."""
    import importlib.util
    spec = importlib.util.spec_from_file_location(
        "h5py_npz", os.path.join(ROOT, "tests", "fixtures", "stubs_h5npz", "h5py", "__init__.py"))
    h5py = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(h5py)
    path = str(tmp_path / "vgg16_pitts_64_desc_cen.hdf5")
    with h5py.File(path, mode="w") as h5:
        feat = h5.create_dataset("descriptors", [10, 4], dtype=np.float32)
        feat[2:4, :] = np.ones((2, 4), np.float32)
        h5.create_dataset("centroids", data=feat[...][:3] * 2)
    assert os.path.isfile(path)
    with h5py.File(path, mode="r") as h5:
        d, c = h5.get("descriptors")[...], h5["centroids"][...]
    assert d.shape == (10, 4) and d.dtype == np.float32 and d[2:4].sum() == 8 and d[:2].sum() == 0
    assert np.array_equal(c, d[:3] * 2)
    assert set(np.load(path).files) == {"descriptors", "centroids"}


def test_vendored_recipe_scripts_are_unmodified():
    pins = {"cluster": "785c1fcf8219c58fdbbb4be5cc7df7013174162b18fe3db7853256f1b0a68452",
            "netvlad_img": "9f2c21800b4cadc563d4e3072dc5b74c193f3133070574391d2429c7e9adbbd5"}
    for script, sha in pins.items():
        data = open(os.path.join(GOLDEN, f"reference_examples_{script}.py.txt"), "rb").read()
        assert hashlib.sha256(data).hexdigest() == sha, script

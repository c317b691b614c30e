"""Host side of the device training transform (`get_transformer_train(h, w, device_decode=True)`): the worker draws
ColorJitter's parameters exactly as the host transform does, and the carriers travel through the repository's tuple
loader.  No GPU needed."""
import ctypes
import os
import pickle
import random

import numpy as np
import pytest
import torch
from PIL import Image


def _pil(h, w, seed):
    return Image.fromarray(np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8))


def test_device_transform_draws_like_color_jitter_and_leaves_the_same_rng_state():
    import torchvision.transforms as T
    from openibl_b200.utils.data import get_transformer_train
    from openibl_b200.utils.data.gpu_jpeg import JitteredImage
    host, dev = get_transformer_train(24, 32), get_transformer_train(24, 32, device_decode=True)
    cj = T.ColorJitter(0.7, 0.7, 0.7, 0.5)
    img = _pil(30, 40, 0)
    for seed in range(300):
        torch.manual_seed(seed)
        order, b, c, s, h = T.ColorJitter.get_params(cj.brightness, cj.contrast, cj.saturation, cj.hue)
        want_state = torch.get_rng_state()
        torch.manual_seed(seed)
        host(img)                                                   # the whole reference transform
        assert torch.equal(torch.get_rng_state(), want_state), seed
        torch.manual_seed(seed)
        got = dev(b"bytes", "f.jpg")
        assert torch.equal(torch.get_rng_state(), want_state), seed
        assert isinstance(got, JitteredImage) and bytes(got) == b"bytes" and got.name == "f.jpg"
        assert (got.height, got.width, got.tokyo) == (24, 32, False)
        assert got.jitter == (tuple(order.tolist()), b, c, s, h), seed


def test_carrier_pickles_with_its_parameters():
    from openibl_b200.utils.data.gpu_jpeg import JitteredImage
    x = JitteredImage(b"\xff\xd8abc", 48, 64, ([3, 1, 0, 2], 0.5, 1.25, None, -0.125), name="a/b.jpg")
    y = pickle.loads(pickle.dumps(x))
    assert type(y) is JitteredImage and bytes(y) == bytes(x)
    assert (y.height, y.width, y.tokyo, y.name, y.jitter) == (48, 64, False, "a/b.jpg", ((3, 1, 0, 2), 0.5, 1.25, None,
                                                                                        -0.125))


class _DrawOnly:
    """The host transform's use of the RNG alone: ColorJitter.get_params, as ColorJitter.forward calls it."""

    def __init__(self):
        import torchvision.transforms as T
        self.cj = T.ColorJitter(0.7, 0.7, 0.7, 0.5)

    def __call__(self, img):
        cj = self.cj
        order, b, c, s, h = cj.get_params(cj.brightness, cj.contrast, cj.saturation, cj.hue)
        return torch.tensor([float(v) for v in order.tolist()] + [b, c, s, h], dtype=torch.float64)


@pytest.fixture(scope="module")
def pitts(tmp_path_factory):
    from openibl_b200 import datasets
    root = str(tmp_path_factory.mktemp("cj_pitts") / "pitts")
    datasets.write_synthetic_pitts_tree(root, scale="30k", n_places=(16, 4, 4), size=(60, 80))
    return datasets.create("pitts", root, scale="30k", verbose=False)


def _tuple_loader(ds, transform, workers, seed):
    from torch.utils.data import DataLoader
    from openibl_b200.utils.data import Preprocessor
    from openibl_b200.utils.data.sampler import DistributedRandomTupleSampler
    s = DistributedRandomTupleSampler(ds.q_train, ds.db_train, ds.train_pos, ds.train_neg, neg_num=3, neg_pool=10,
                                      num_replicas=1, rank=0)
    rng = np.random.default_rng(1)
    s.sort_idx = torch.from_numpy(np.stack([rng.permutation(len(ds.db_train)) for _ in ds.q_train]))
    pre = Preprocessor(ds.q_train + ds.db_train, root=ds.images_dir, transform=transform)
    random.seed(seed)
    torch.manual_seed(seed)
    dl = DataLoader(pre, batch_size=2, num_workers=workers, sampler=s, shuffle=False, pin_memory=False, drop_last=True)
    return list(dl)


@pytest.mark.parametrize("workers", [0, 2])
def test_carriers_collate_through_the_tuple_loader(pitts, workers):
    from openibl_b200.utils.data import get_transformer_train
    from openibl_b200.utils.data.gpu_jpeg import JitteredImage, is_encoded_batch
    dev = _tuple_loader(pitts, get_transformer_train(60, 80, device_decode=True), workers, 7)
    draws = _tuple_loader(pitts, _DrawOnly(), workers, 7)
    assert len(dev) == len(draws) > 0
    for batch, ref in zip(dev, draws):
        assert len(batch) == 5                                     # anchor, positive, 3 negatives
        for pos, rpos in zip(batch, ref):
            carriers, fnames = pos[0], pos[1]
            assert is_encoded_batch(carriers) and all(type(x) is JitteredImage for x in carriers)
            assert list(fnames) == list(rpos[1])
            for x, fname, want in zip(carriers, fnames, rpos[0]):
                assert x.name == fname
                with open(os.path.join(pitts.images_dir, fname), "rb") as f:
                    assert bytes(x) == f.read()
                order, b, c, s, h = x.jitter
                assert torch.equal(torch.tensor([float(v) for v in order] + [b, c, s, h], dtype=torch.float64), want)


def test_library_exports_color_jitter():
    from openibl_b200 import _cabi
    lib = ctypes.CDLL(_cabi.LIB_PATH)
    assert hasattr(lib, "ibl_color_jitter_u8")
    assert "ibl_color_jitter_u8" in _cabi.SIGNATURES

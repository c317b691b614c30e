"""Device colour jitter (csrc/color_jitter.cu) and the training loader's file-bytes path: bit-exact against
torchvision's PIL transforms run in the same test, and trainer inputs identical to the host loader's."""
import io
import random

import numpy as np
import pytest
import torch
from PIL import Image

pytestmark = pytest.mark.gpu

OPS = ("brightness", "contrast", "saturation", "hue")


@pytest.fixture(scope="module")
def eng():
    from openibl_b200.engine import Engine
    return Engine.get(0)


def _jitter(eng, arrays, params):
    """Jitter host uint8 HWC arrays as views into one device buffer (the decoder's layout)."""
    flat = torch.cat([torch.from_numpy(np.array(a)).reshape(-1) for a in arrays]).cuda()
    views = [v.view(a.shape) for v, a in zip(flat.split([a.size for a in arrays]), arrays)]
    eng.color_jitter_u8(views, params)
    return [v.cpu().numpy() for v in views]


def _diff(got, want, what):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if not np.array_equal(got, want):
        d = np.argwhere(got != want)
        raise AssertionError(f"{what}: {len(d)} bytes differ, first at {d[0].tolist()}: "
                             f"got {got[tuple(d[0][:2])]} want {want[tuple(d[0][:2])]}")


@pytest.fixture(scope="module")
def all_colours():
    c = np.arange(256, dtype=np.uint8)
    return np.stack(np.meshgrid(c, c, c, indexing="ij"), -1).reshape(4096, 4096, 3)


@pytest.mark.parametrize("op", OPS)
def test_each_op_alone_on_all_colours(eng, all_colours, op):
    import torchvision.transforms.functional as F
    fn = {"brightness": F.adjust_brightness, "contrast": F.adjust_contrast, "saturation": F.adjust_saturation,
          "hue": F.adjust_hue}[op]
    factors = (-0.5, -0.1, 0.0, 0.002, 0.5) if op == "hue" else (0.3, 1.0, 1.7)
    pil = Image.fromarray(all_colours)
    for f in factors:
        want = np.asarray(fn(pil, f))
        params = [None] * 4
        params[OPS.index(op)] = f
        got, = _jitter(eng, [all_colours], [((0, 1, 2, 3), *params)])
        _diff(got, want, f"{op} {f}")


def _image(kind, h, w, rng):
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "uniform":
        return np.broadcast_to(rng.integers(0, 256, 3, dtype=np.uint8), (h, w, 3)).copy()
    base = rng.integers(0, 256, (h // 16 + 2, w // 16 + 2, 3)).astype(np.uint8)
    a = np.asarray(Image.fromarray(base).resize((w, h), Image.BILINEAR))
    return np.repeat(a[..., :1], 3, -1) if kind == "grey" else a


SIZES = [(1, 1), (7, 9), (480, 640), (481, 643), (1224, 1632)]
KINDS = ("noise", "smooth", "grey", "uniform")


def test_seeded_color_jitter_draws_mixed_sizes(eng):
    import torchvision.transforms as T
    cj = T.ColorJitter(0.7, 0.7, 0.7, 0.5)
    rng = np.random.default_rng(0)
    for call in range(44):                                    # 220 draws, five sizes per call, kinds rotate
        arrays, params, wants = [], [], []
        for j, (h, w) in enumerate(SIZES):
            k = call * len(SIZES) + j
            a = _image(KINDS[call % len(KINDS)], h, w, rng)
            torch.manual_seed(k)
            wants.append(np.asarray(cj(Image.fromarray(a))))
            torch.manual_seed(k)
            order, b, c, s, hue = T.ColorJitter.get_params(cj.brightness, cj.contrast, cj.saturation, cj.hue)
            arrays.append(a)
            params.append((order.tolist(), b, c, s, hue))
        for a, p, g, want in zip(arrays, params, _jitter(eng, arrays, params), wants):
            _diff(g, want, f"call {call} {KINDS[call % len(KINDS)]} {a.shape} {p}")


def _jpeg(h, w, seed, mode="RGB", **kw):
    rng = np.random.default_rng(seed)
    im = Image.fromarray(_image("smooth", h, w, rng))
    b = io.BytesIO()
    (im.convert("L") if mode == "L" else im).save(b, "JPEG", quality=92, **kw)
    return b.getvalue()


def test_decode_to_tensor_with_jitter_matches_host_train_transform(eng):
    from openibl_b200.utils.data import get_transformer_train
    from openibl_b200.utils.data.gpu_jpeg import decode_batch
    files = [_jpeg(480, 640, 1), _jpeg(480, 640, 2, progressive=True), _jpeg(480, 640, 3, "L"),
             _jpeg(300, 400, 4, subsampling=1), _jpeg(481, 643, 5)]
    for h, w in ((480, 640), (240, 320)):
        host, dev = get_transformer_train(h, w), get_transformer_train(h, w, device_decode=True)
        want, carriers = [], []
        for i, f in enumerate(files):
            torch.manual_seed(50 + i)
            want.append(host(Image.open(io.BytesIO(f)).convert("RGB")))
            torch.manual_seed(50 + i)
            carriers.append(dev(f, f"f{i}.jpg"))
        got = decode_batch(carriers).cpu()
        for i in range(len(files)):
            assert torch.equal(got[i], want[i]), (h, w, i, (got[i] - want[i]).abs().max())


def test_host_fallback_shares_the_decode_buffer_and_jitter_needs_one_buffer(eng):
    from openibl_b200.utils.data.gpu_jpeg import _host_decode
    files = [_jpeg(48, 64, 6), _jpeg(40, 56, 7, progressive=True), _jpeg(48, 64, 8)]
    imgs, _ = eng.decode_jpeg_async(files, fallback=_host_decode)
    assert len({im.untyped_storage().data_ptr() for im in imgs}) == 1
    assert np.array_equal(imgs[1].cpu().numpy(), _host_decode(files[1]))
    apart = [im.clone() for im in imgs]
    with pytest.raises(ValueError, match="one device buffer"):
        eng.color_jitter_u8(apart, [((0, 1, 2, 3), 0.5, None, None, None)] * 3)


@pytest.fixture(scope="module")
def pitts(tmp_path_factory):
    from openibl_b200 import datasets
    root = str(tmp_path_factory.mktemp("cj_train") / "pitts")
    datasets.write_synthetic_pitts_tree(root, scale="30k", n_places=(16, 4, 4))
    return datasets.create("pitts", root, scale="30k", verbose=False)


def _loader(ds, device_decode, workers, diff, seed=5):
    from torch.utils.data import DataLoader
    from openibl_b200.utils.data import Preprocessor, get_transformer_train
    from openibl_b200.utils.data.sampler import DistributedRandomDiffTupleSampler, DistributedRandomTupleSampler
    nq, ng = len(ds.q_train), len(ds.db_train)
    if diff:
        # one difficult positive: tuples of one length, so the default collate stacks them at batch size 2
        s = DistributedRandomDiffTupleSampler(ds.q_train, ds.db_train, ds.train_pos, ds.train_neg, pos_num=1,
                                              pos_pool=4, neg_num=3, neg_pool=10, num_replicas=1, rank=0)
        s.distmat_jac = torch.from_numpy(np.random.default_rng(2).random((nq, ng)).astype(np.float32))
    else:
        s = DistributedRandomTupleSampler(ds.q_train, ds.db_train, ds.train_pos, ds.train_neg, neg_num=3,
                                          neg_pool=10, num_replicas=1, rank=0)
    rng = np.random.default_rng(1)
    s.sort_idx = torch.from_numpy(np.stack([rng.permutation(ng) for _ in range(nq)]))
    pre = Preprocessor(ds.q_train + ds.db_train, root=ds.images_dir,
                       transform=get_transformer_train(96, 128, device_decode=device_decode))
    random.seed(seed)
    torch.manual_seed(seed)
    return list(DataLoader(pre, batch_size=2, num_workers=workers, sampler=s, shuffle=False, pin_memory=True,
                           drop_last=True))


def _model():
    from openibl_b200 import models, synth
    torch.manual_seed(3)
    base = models.create("vgg16", pretrained=False)
    pool = models.create("netvlad", dim=base.feature_dim)
    p = synth.make_netvlad_params(seed=3, sharp=True)
    pool.centroids.data.copy_(p["centroids"])
    pool.conv.weight.data.copy_(p["conv_weight"])
    return models.create("embednet", base, pool).cuda()


@pytest.mark.parametrize("workers", [0, 2])
def test_trainer_inputs_and_loss_identical_with_device_decode(pitts, workers):
    from openibl_b200.trainers import Trainer
    host, dev = _loader(pitts, False, workers, False), _loader(pitts, True, workers, False)
    assert len(host) == len(dev) > 0
    model = _model()
    model.train()
    tr = Trainer(model, margin=0.1, gpu=0)
    for i, (hb, db) in enumerate(zip(host, dev)):
        x_host, x_dev = tr._parse_data(hb), tr._parse_data(db)
        assert x_dev.shape == x_host.shape == (2, 5, 3, 96, 128) and x_dev.is_cuda
        assert torch.equal(x_host, x_dev), i
    loss_host = tr._forward(x_host, True, "triplet")
    loss_dev = tr._forward(x_dev, True, "triplet")
    assert torch.isfinite(loss_host) and torch.equal(loss_host, loss_dev)


@pytest.mark.parametrize("workers", [0, 2])
def test_sfrs_trainer_inputs_identical_with_device_decode(pitts, workers):
    from openibl_b200.trainers import SFRSTrainer
    host, dev = _loader(pitts, False, workers, True), _loader(pitts, True, workers, True)
    assert len(host) == len(dev) > 0
    tr = SFRSTrainer(None, None, neg_num=3, gpu=0)
    for i, (hb, db) in enumerate(zip(host, dev)):
        (he, hd), (de, dd) = tr._parse_data(hb), tr._parse_data(db)
        assert de.shape == he.shape == (2, 5, 3, 96, 128) and dd.shape == hd.shape == (2, 2, 3, 96, 128)
        assert torch.equal(he, de) and torch.equal(hd, dd), i


def test_corrupt_file_in_training_tuple_raises_naming_it(eng):
    from openibl_b200.trainers import Trainer
    from openibl_b200.utils.data import get_transformer_train
    good = _jpeg(96, 128, 21)
    sos = good.index(b"\xff\xda")
    start = sos + 2 + int.from_bytes(good[sos + 2: sos + 4], "big")
    mid = (start + len(good)) // 2
    bad = good[:mid] + b"\xff\x00" * 64 + good[mid + 128:]        # 512 one-bits: no codeword starts with 16 ones
    tf = get_transformer_train(96, 128, device_decode=True)
    names = [[f"t{b}_p{n}.jpg" for b in range(2)] for n in range(3)]
    inputs = [[[tf(bad if (b, n) == (1, 2) else good, names[n][b]) for b in range(2)], names[n]] for n in range(3)]
    with pytest.raises(RuntimeError, match="t1_p2.jpg"):
        Trainer(None, gpu=0)._parse_data(inputs)
    torch.cuda.synchronize()

"""Device JPEG decode (csrc/jpeg.cu) and the file-bytes loader path: bit-exact against Pillow's decode of the same
bytes, and descriptors / recalls identical to the host transform path."""
import io
import os

import numpy as np
import pytest
import torch
from PIL import Image

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from openibl_b200.engine import Engine
    return Engine.get(0)


def _img(h, w, seed, mode="RGB", noise=False):
    r = np.random.default_rng(seed)
    if noise:
        a = r.integers(0, 256, (h, w, 3), dtype=np.uint8)
    else:
        base = r.integers(0, 256, (h // 8 + 2, w // 8 + 2, 3)).astype(np.uint8)
        a = np.asarray(Image.fromarray(base).resize((w, h), Image.BILINEAR)).astype(np.int16)
        a = np.clip(a + r.integers(-20, 21, a.shape), 0, 255).astype(np.uint8)
    im = Image.fromarray(a)
    return im.convert("L") if mode == "L" else im


def _jpeg(im, **kw):
    b = io.BytesIO()
    im.save(b, "JPEG", **kw)
    return b.getvalue()


def _pil(data):
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


def _check(eng, files):
    got = eng.decode_jpeg(files)
    torch.cuda.synchronize()
    for i, (g, f) in enumerate(zip(got, files)):
        assert g is not None, i
        want = _pil(f)
        g = g.cpu().numpy()
        assert g.shape == want.shape, (i, g.shape, want.shape)
        if not np.array_equal(g, want):
            d = np.argwhere(g != want)
            raise AssertionError(f"file {i}: {len(d)} bytes differ, first at {d[0].tolist()}")


SIZES = [(1, 1), (7, 9), (17, 33), (480, 640), (481, 643), (1224, 1632), (4003, 21)]


@pytest.mark.parametrize("sub", [0, 1, 2, "L"])
def test_decode_bit_exact_sizes_and_sampling(eng, sub):
    mode = "L" if sub == "L" else "RGB"
    kw = {} if sub == "L" else {"subsampling": sub}
    files = [_jpeg(_img(h, w, h + w, mode), quality=92, **kw) for h, w in SIZES]
    _check(eng, files)                                         # one mixed-size batch


@pytest.mark.parametrize("quality", [50, 75, 92, 100])
def test_decode_bit_exact_quality_optimize_restart(eng, quality):
    im = _img(240, 328, quality)
    files = [_jpeg(im, quality=quality, subsampling=s) for s in (0, 1, 2)]
    files += [_jpeg(im, quality=quality, optimize=True), _jpeg(im, quality=quality, restart_marker_blocks=5),
              _jpeg(im, quality=quality, restart_marker_rows=1, subsampling=0),
              _jpeg(im.convert("L"), quality=quality, restart_marker_blocks=3)]
    _check(eng, files)


def test_decode_bit_exact_high_entropy(eng):
    files = [_jpeg(_img(480, 640, 3, noise=True), quality=100, subsampling=0),
             _jpeg(_img(333, 517, 4, noise=True), quality=92, subsampling=2)]
    _check(eng, files)


def test_decode_to_tensor_matches_host_transform_and_falls_back(eng):
    from openibl_b200.utils.data import get_transformer_test
    from openibl_b200.utils.data.gpu_jpeg import decode_to_tensor
    files = [_jpeg(_img(480, 640, 11), quality=92), _jpeg(_img(480, 640, 12), quality=92, progressive=True),
             _jpeg(_img(300, 400, 13), quality=75, subsampling=1), _jpeg(_img(480, 640, 14, "L"), quality=92)]
    for h, w in ((480, 640), (240, 320)):
        tf = get_transformer_test(h, w)
        want = torch.stack([tf(Image.open(io.BytesIO(f)).convert("RGB")) for f in files])
        got = decode_to_tensor(files, h, w).cpu()
        assert torch.equal(got, want), (h, w, (got - want).abs().max())
    # Tokyo: T.Resize(max(h, w)) from each image's own size (batch of one, as the reference's Tokyo loaders)
    tf = get_transformer_test(480, 640, tokyo=True)
    for f in (files[0], files[2], _jpeg(_img(640, 480, 15), quality=92)):
        want = tf(Image.open(io.BytesIO(f)).convert("RGB")).unsqueeze(0)
        got = decode_to_tensor([f], 480, 640, tokyo=True).cpu()
        assert torch.equal(got, want)


def test_corrupt_entropy_data_raises_naming_the_file(eng):
    from openibl_b200.utils.data.gpu_jpeg import EncodedImage, decode_batch
    good = _jpeg(_img(96, 128, 21), quality=92)
    sos = good.index(b"\xff\xda")
    start = sos + 2 + int.from_bytes(good[sos + 2: sos + 4], "big")
    mid = (start + len(good)) // 2
    # 512 one-bits (stuffed 0xFF 0x00 pairs) inside the scan: no codeword starts with 16 ones
    bad = good[:mid] + b"\xff\x00" * 64 + good[mid + 128:]
    batch = [EncodedImage(good, 96, 128, name="ok.jpg"), EncodedImage(bad, 96, 128, name="broken.jpg")]
    with pytest.raises(RuntimeError, match="broken.jpg"):
        decode_batch(batch)
    torch.cuda.synchronize()
    _check(eng, [good])                                        # the process and the engine carry on


def _model(pca_dim=None):
    from openibl_b200 import models, synth
    torch.manual_seed(3)
    base = models.create("vgg16", pretrained=False)
    pool = models.create("netvlad", dim=base.feature_dim)
    p = synth.make_netvlad_params(seed=3, sharp=True)
    pool.centroids.data.copy_(p["centroids"])
    pool.conv.weight.data.copy_(p["conv_weight"])
    if pca_dim:
        return models.create("embednetpca", base, pool, dim=pca_dim).cuda()
    return models.create("embednet", base, pool).cuda()


@pytest.fixture(scope="module")
def pitts(tmp_path_factory):
    from openibl_b200 import datasets
    root = str(tmp_path_factory.mktemp("jpeg_pitts") / "pitts")
    datasets.write_synthetic_pitts_tree(root, scale="30k")
    return datasets.create("pitts", root, scale="30k", verbose=False)


def _loader(ds, items, device_decode, h=96, w=128):
    from torch.utils.data import DataLoader
    from openibl_b200.utils.data import Preprocessor, get_transformer_test
    pre = Preprocessor(items, root=ds.images_dir, transform=get_transformer_test(h, w, device_decode=device_decode))
    return DataLoader(pre, batch_size=8, num_workers=2, shuffle=False, pin_memory=True)


@pytest.mark.parametrize("pca_dim", [None, 64])
def test_extract_features_identical_with_device_decode(pitts, pca_dim):
    from openibl_b200.evaluators import extract_features
    model = _model(pca_dim)
    items = sorted(list(set(pitts.q_test) | set(pitts.db_test)))
    host = extract_features(model, _loader(pitts, items, False), items, print_freq=1000)
    dev = extract_features(model, _loader(pitts, items, True), items, print_freq=1000)
    assert list(host) == list(dev)
    for k in host:
        assert torch.equal(host[k], dev[k]), k


def test_evaluator_recalls_identical_with_device_decode(pitts):
    from openibl_b200.evaluators import Evaluator
    model = _model()
    ev = Evaluator(model)
    dataset = sorted(list(set(pitts.q_test) | set(pitts.db_test)))
    rec = []
    for dd in (False, True):
        rec.append(ev.evaluate(_loader(pitts, pitts.q_test, dd), dataset, pitts.q_test, pitts.db_test, pitts.test_pos,
                               gallery_loader=_loader(pitts, pitts.db_test, dd), vlad=True))
    assert np.array_equal(np.asarray(rec[0]), np.asarray(rec[1])), rec
    assert 0 < rec[0][0] <= 1

"""Device decode of progressive JPEGs (csrc/jpeg.cu, ibl_jpeg_decode_progressive_u8): bit-exact against Pillow's
decode of the same bytes, sharing one buffer with baseline and host-decoded files, and the loader paths unchanged in
their results when a dataset is progressive."""
import io
import os

import numpy as np
import pytest
import torch
from PIL import Image, ImageFile

from test_host_jpeg_progressive import custom_script_files

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
    # with `progressive` Pillow's encoder needs the whole file to fit its output buffer, max(MAXBLOCK, w * h) bytes,
    # which high-entropy images overflow
    old = ImageFile.MAXBLOCK
    ImageFile.MAXBLOCK = max(old, 8 * im.size[0] * im.size[1])
    try:
        b = io.BytesIO()
        im.save(b, "JPEG", **kw)
        return b.getvalue()
    finally:
        ImageFile.MAXBLOCK = old


def _pil(data):
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


def _check(eng, files):
    from openibl_b200 import _cabi
    for i, f in enumerate(files):
        assert _cabi.jpeg_parse_progressive(f)["ok"], (i, _cabi.jpeg_parse_progressive(f)["reason"])
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
def test_progressive_bit_exact_sizes_and_sampling(eng, sub):
    mode = "L" if sub == "L" else "RGB"
    kw = {} if sub == "L" else {"subsampling": sub}
    files = [_jpeg(_img(h, w, h + w, mode), quality=92, progressive=True, **kw) for h, w in SIZES]
    _check(eng, files)


@pytest.mark.parametrize("quality", [50, 75, 92, 100])
def test_progressive_bit_exact_quality_optimize_restart(eng, quality):
    im = _img(240, 328, quality)
    files = [_jpeg(im, quality=quality, subsampling=s, progressive=True) for s in (0, 1, 2)]
    files += [_jpeg(im, quality=quality, optimize=True, progressive=True),
              _jpeg(im, quality=quality, restart_marker_blocks=5, progressive=True),
              _jpeg(im, quality=quality, restart_marker_rows=1, subsampling=0, progressive=True),
              _jpeg(im.convert("L"), quality=quality, restart_marker_blocks=3, progressive=True),
              _jpeg(im.convert("L"), quality=quality, optimize=True, progressive=True)]
    _check(eng, files)


def test_progressive_bit_exact_high_entropy(eng):
    files = [_jpeg(_img(480, 640, 3, noise=True), quality=100, subsampling=0, progressive=True),
             _jpeg(_img(333, 517, 4, noise=True), quality=92, subsampling=2, progressive=True),
             _jpeg(_img(129, 77, 5, noise=True), quality=75, subsampling=1, progressive=True, restart_marker_blocks=2)]
    _check(eng, files)


def test_progressive_bit_exact_custom_scan_scripts(eng):
    """Scripts Pillow cannot write: spectral selection only, non-interleaved DC, no DC successive approximation,
    long end-of-band runs, Huffman tables redefined before every scan, restart intervals."""
    files = [f for _, f in custom_script_files()]
    _check(eng, files)


def test_mixed_batch_shares_one_buffer_and_pillow_sees_only_the_rest(eng, monkeypatch):
    from openibl_b200.utils.data import gpu_jpeg
    im = _img(120, 160, 31)
    files = [_jpeg(im, quality=90), _jpeg(im, quality=90, progressive=True), _jpeg(im.convert("CMYK"), quality=90),
             _jpeg(_img(64, 48, 32, "L"), quality=80, progressive=True), _jpeg(_img(33, 65, 33), quality=85)]
    seen = []
    real = gpu_jpeg._host_decode

    def spy(data):
        seen.append(bytes(data))
        return real(data)
    monkeypatch.setattr(gpu_jpeg, "_host_decode", spy)
    imgs, err = eng.decode_jpeg_async(files, fallback=gpu_jpeg._host_decode)
    torch.cuda.synchronize()
    assert seen == [files[2]]
    base = imgs[0].untyped_storage().data_ptr()
    assert all(x.untyped_storage().data_ptr() == base for x in imgs)
    assert not err.any()
    for g, f in zip(imgs, files):
        assert np.array_equal(g.cpu().numpy(), _pil(f))
    # without a fallback the progressive files come back too; only the CMYK file is None
    got = eng.decode_jpeg(files)
    assert [g is None for g in got] == [False, False, True, False, False]


def test_jitter_path_with_progressive_files_matches_host_train_transform(eng):
    from openibl_b200.utils.data import get_transformer_train
    from openibl_b200.utils.data.gpu_jpeg import decode_batch
    files = [_jpeg(_img(480, 640, 41), quality=92, progressive=True),
             _jpeg(_img(480, 640, 42, "L"), quality=92, progressive=True),
             _jpeg(_img(300, 400, 43), quality=75, subsampling=1, progressive=True),
             _jpeg(_img(480, 640, 44), quality=92)]
    for h, w in ((480, 640), (240, 320)):
        host, dev = get_transformer_train(h, w), get_transformer_train(h, w, device_decode=True)
        want, carriers = [], []
        for i, f in enumerate(files):
            torch.manual_seed(70 + i)
            want.append(host(Image.open(io.BytesIO(f)).convert("RGB")))
            torch.manual_seed(70 + i)
            carriers.append(dev(f, f"p{i}.jpg"))
        got = decode_batch(carriers).cpu()
        for i in range(len(files)):
            assert torch.equal(got[i], want[i]), (h, w, i, (got[i] - want[i]).abs().max())


def _scan_payload(data, k):
    """(start, end) of the entropy-coded bytes of scan k."""
    pos = -1
    for _ in range(k + 1):
        pos = data.index(b"\xff\xda", pos + 1)
    start = pos + 2 + int.from_bytes(data[pos + 2: pos + 4], "big")
    end = start
    while not (data[end] == 0xFF and data[end + 1] not in (0x00,) and not 0xD0 <= data[end + 1] <= 0xD7):
        end += 1
    return start, end


@pytest.mark.parametrize("scan", [0, 1, 5, 9])
def test_corrupt_progressive_stream_raises_naming_the_file(eng, scan):
    from openibl_b200.utils.data.gpu_jpeg import EncodedImage, decode_batch
    good = _jpeg(_img(96, 128, 51), quality=92, progressive=True)
    start, end = _scan_payload(good, scan)
    # cut the scan's data short: the interval ends before its last block
    bad = good[:start] + good[start: start + max(1, (end - start) // 4)] + good[end:]
    batch = [EncodedImage(good, 96, 128, name="ok.jpg"), EncodedImage(bad, 96, 128, name="broken.jpg")]
    with pytest.raises(RuntimeError, match="broken.jpg"):
        decode_batch(batch)
    torch.cuda.synchronize()
    _check(eng, [good])                                        # the process and the engine carry on


def test_invalid_code_in_progressive_scan_raises(eng):
    from openibl_b200.utils.data.gpu_jpeg import EncodedImage, decode_batch
    good = _jpeg(_img(96, 128, 52), quality=92, progressive=True)
    start, end = _scan_payload(good, 1)
    mid = (start + end) // 2
    bad = good[:mid] + b"\xff\x00" * 8 + good[mid + 16:]      # 64 one-bits: no codeword starts with 16 ones
    with pytest.raises(RuntimeError, match="broken.jpg"):
        decode_batch([EncodedImage(bad, 96, 128, name="broken.jpg")])
    torch.cuda.synchronize()


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
    """The synthetic Pittsburgh tree with every image re-saved as a progressive JPEG."""
    from openibl_b200 import datasets
    root = str(tmp_path_factory.mktemp("jpeg_prog_pitts") / "pitts")
    datasets.write_synthetic_pitts_tree(root, scale="30k")
    n = 0
    for d, _, names in os.walk(root):
        for name in names:
            if name.endswith(".jpg"):
                p = os.path.join(d, name)
                im = Image.open(p).convert("RGB")
                im.save(p, "JPEG", quality=90, progressive=True)
                n += 1
    assert n > 0
    return datasets.create("pitts", root, scale="30k", verbose=False)


def _loader(ds, items, device_decode, h=96, w=128):
    from torch.utils.data import DataLoader
    from openibl_b200.utils.data import Preprocessor, get_transformer_test
    pre = Preprocessor(items, root=ds.images_dir, transform=get_transformer_test(h, w, device_decode=device_decode))
    return DataLoader(pre, batch_size=8, num_workers=2, shuffle=False, pin_memory=True)


def test_progressive_dataset_is_decoded_on_the_device(pitts, monkeypatch):
    from openibl_b200.utils.data import gpu_jpeg
    items = sorted(list(set(pitts.q_test) | set(pitts.db_test)))[:8]
    files = [open(os.path.join(pitts.images_dir, it[0]), "rb").read() for it in items]

    def refuse(data):
        raise AssertionError("a progressive file reached the host decoder")
    monkeypatch.setattr(gpu_jpeg, "_host_decode", refuse)
    gpu_jpeg.decode_to_tensor(files, 96, 128)


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

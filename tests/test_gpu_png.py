"""Device decode of PNGs (csrc/png.cu, ibl_png_decode_u8): bit-exact against Pillow's decode of the same bytes over
colour types, sizes, filters, zlib strategies and IDAT splits; the acceptance table; one buffer shared with JPEGs and
host-decoded files; and the loader paths unchanged in their results on a Tokyo-shaped dataset whose database is PNG."""
import io
import json
import os
import shutil
import zlib

import numpy as np
import pytest
import torch
from PIL import Image

from test_host_png import BPP, STRATEGIES, corrupt_cases, far_match_cinfo1, huffman_cases, image, parse, pillow, png_file

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from openibl_b200.engine import Engine
    return Engine.get(0)


def _pal(seed, n=256):
    return np.random.default_rng(seed).integers(0, 256, (n, 3))


def _check(eng, files):
    for i, f in enumerate(files):
        assert parse(f)["ok"], (i, parse(f)["reason"])
    got = eng.decode_jpeg(files)
    torch.cuda.synchronize()
    for i, (g, f) in enumerate(zip(got, files)):
        assert g is not None, i
        want = pillow(f)
        g = g.cpu().numpy()
        assert g.shape == want.shape, (i, g.shape, want.shape)
        if not np.array_equal(g, want):
            d = np.argwhere(g != want)
            raise AssertionError(f"file {i}: {len(d)} bytes differ, first at {d[0].tolist()}")


SIZES = [(1, 1), (1, 37), (29, 1), (97, 131), (300, 7), (480, 640)]


@pytest.mark.parametrize("ct", [0, 2, 3, 4, 6])
def test_png_bit_exact_colour_types_sizes_filters(eng, ct):
    files = []
    for k, (h, w) in enumerate(SIZES):
        a = image(h, w, ct, 100 * ct + k, noise=k % 2 == 1)
        for filters in ((0,), (1,), (2,), (3,), (4,), (0, 1, 2, 3, 4)):
            if (h, w) == (480, 640) and len(filters) == 1 and filters[0] in (0, 2):
                continue
            files.append(png_file(a, ct, filters=filters, palette=_pal(ct) if ct == 3 else None))
    _check(eng, files)


def test_png_bit_exact_pillow_encoder(eng):
    files = []
    for k, mode in enumerate(("RGB", "L", "RGBA", "LA", "P")):
        for h, w in ((480, 640), (97, 131), (1, 1)):
            im = Image.fromarray(image(h, w, 2, 7 + k)).convert(mode)
            for opt in ({}, {"optimize": True}, {"compress_level": 1}, {"compress_level": 9}):
                b = io.BytesIO()
                im.save(b, "PNG", **opt)
                files.append(b.getvalue())
    _check(eng, files)


@pytest.mark.parametrize("level,strategy", STRATEGIES)
def test_png_bit_exact_zlib_strategies_and_idat_splits(eng, level, strategy):
    a = image(120, 160, 2, level + 10 * strategy)
    files = [png_file(a, 2, level=level, strategy=strategy, split=s) for s in (None, 1, 7, 1000, 8192)]
    noise = image(64, 96, 6, 3, noise=True)
    files.append(png_file(noise, 6, level=level, strategy=strategy))
    _check(eng, files)


def test_png_small_window_and_far_matches(eng):
    # CINFO < 7 headers, and 258-byte matches at distance 32768: a 32 KiB noise row block repeated
    h, w = 64, 1024
    base = np.random.default_rng(5).integers(0, 256, (h // 2, w, 1), dtype=np.uint8)
    a = np.concatenate([base, base])
    files = [png_file(a, 0, filters=(0,), level=9),
             png_file(image(80, 90, 2, 6), 2, wbits=9), png_file(image(80, 90, 2, 7), 2, wbits=12, level=1)]
    assert files[1][files[1].index(b"IDAT") + 4] >> 4 == 1
    _check(eng, files)


def test_png_cinfo_below_7_with_far_matches(eng):
    a, z = far_match_cinfo1()
    _check(eng, [png_file(a, 0, zlib_stream=z)])


def test_code_sets_follow_zlib(eng):
    """Valid single-code and empty distance codes decode; over-subscribed and incomplete codes, a missing end-of-block
    code and a distance past the output set the data error (1) even though the rows are already complete."""
    cases = huffman_cases()
    files = [png_file(np.zeros((1, 4, 1), np.uint8), 0, zlib_stream=z) for z, _ in cases.values()]
    imgs, err = eng.decode_jpeg_async(files)
    torch.cuda.synchronize()
    for (name, (_, ok)), f, im, e in zip(cases.items(), files, imgs, err.cpu().tolist()):
        if ok:
            assert e == 0, name
            assert np.array_equal(im.cpu().numpy(), pillow(f)), name
        else:
            assert e == 1, (name, e)


def test_png_short_palette_and_trns(eng):
    a = np.random.default_rng(8).integers(0, 9, (17, 23, 1), dtype=np.uint8)
    files = [png_file(a, 3, palette=_pal(1, 5)), png_file(a, 3, palette=_pal(2, 9), trns=b"\x00\x80\xff"),
             png_file(image(9, 9, 0, 1), 0, trns=b"\x00\x07"), png_file(image(9, 9, 2, 1), 2, trns=b"\x00\x01" * 3)]
    _check(eng, files)


def test_acceptance_table(eng):
    from openibl_b200.utils.data.gpu_jpeg import EncodedImage, decode_batch
    for name, (f, pil, dev) in corrupt_cases().items():
        p = parse(f)
        if dev == "reject":
            assert not p["ok"], name
            continue
        assert p["ok"], (name, p["reason"])
        imgs, err = eng.decode_jpeg_async([f])
        torch.cuda.synchronize()
        if dev == "ok":
            assert int(err[0]) == 0, (name, int(err[0]))
            assert np.array_equal(imgs[0].cpu().numpy(), pillow(f)), name
        else:
            assert int(err[0]) != 0, name
            h, w = p["height"], p["width"]
            with pytest.raises(RuntimeError, match=r"PNG.*broken\.png"):
                decode_batch([EncodedImage(f, h, w, name="broken.png")])
    _check(eng, [png_file(image(30, 40, 2, 1), 2)])                 # the engine carries on


def test_corrupt_deflate_streams_set_the_error_word(eng):
    a = image(40, 50, 2, 11)
    bad = []
    for k, pattern in enumerate((b"\xff" * 6, b"\x00" * 6, b"\x5a\xa5" * 3)):
        z = bytearray(zlib.compress(_rows(a, 2), 6))
        mid = len(z) // 3 + k
        z[mid: mid + len(pattern)] = pattern
        bad.append(png_file(a, 2, zlib_stream=bytes(z)))
    bad.append(png_file(a, 2, zlib_stream=b"\x78\x9c" + bytes([0b111]) + b"\0" * 20))         # block type 3
    bad.append(png_file(a, 2, zlib_stream=b"\x78\x9c\x01\x05\x00\x00\x00" + b"\0" * 20))     # LEN != ~NLEN
    _, err = eng.decode_jpeg_async(bad)
    torch.cuda.synchronize()
    assert all(int(e) != 0 for e in err.cpu()), err


def _rows(a, ct):
    from test_host_png import filter_rows
    h, w = a.shape[:2]
    return filter_rows(a.reshape(h, w * BPP[ct]), [0, 1, 2, 3, 4], BPP[ct])


def _jpeg(a, **kw):
    b = io.BytesIO()
    Image.fromarray(a).save(b, "JPEG", **kw)
    return b.getvalue()


def test_mixed_batch_shares_one_buffer_and_pillow_sees_only_the_rest(eng, monkeypatch):
    from openibl_b200.utils.data import gpu_jpeg
    a = image(120, 160, 2, 31)
    b16 = io.BytesIO()
    Image.fromarray(image(40, 50, 0, 3)[..., 0].astype(np.uint16) * 257).save(b16, "PNG")
    files = [_jpeg(a, quality=90), _jpeg(a, quality=90, progressive=True), png_file(a, 2), b16.getvalue(),
             png_file(image(33, 65, 3, 2), 3, palette=_pal(3)), png_file(image(64, 48, 4, 4), 4)]
    assert not parse(files[3])["ok"] and parse(files[3])["reason"] == "bit depth is not 8"
    seen = []
    real = gpu_jpeg._host_decode

    def spy(data):
        seen.append(bytes(data))
        return real(data)
    monkeypatch.setattr(gpu_jpeg, "_host_decode", spy)
    imgs, err = eng.decode_jpeg_async(files, fallback=gpu_jpeg._host_decode)
    torch.cuda.synchronize()
    assert seen == [files[3]]
    base = imgs[0].untyped_storage().data_ptr()
    assert all(x.untyped_storage().data_ptr() == base for x in imgs)
    assert not err.any()
    for g, f in zip(imgs, files):
        assert np.array_equal(g.cpu().numpy(), pillow(f))
    got = eng.decode_jpeg(files)
    assert [g is None for g in got] == [False, False, False, True, False, False]


@pytest.mark.parametrize("tokyo", [False, True])
def test_decode_to_tensor_matches_host_transform(eng, tokyo):
    from openibl_b200.utils.data import get_transformer_test
    from openibl_b200.utils.data.gpu_jpeg import decode_to_tensor
    sizes = [(480, 640)] if tokyo else [(480, 640), (240, 320)]
    a = image(480, 640, 2, 21)
    files = [png_file(a, 2), png_file(image(480, 640, 0, 22), 0), png_file(image(480, 640, 6, 23), 6)]
    for h, w in sizes:
        host = get_transformer_test(h, w, tokyo=tokyo)
        want = torch.stack([host(Image.open(io.BytesIO(f)).convert("RGB")) for f in files])
        got = decode_to_tensor(files, h, w, tokyo=tokyo).cpu()
        assert torch.equal(got, want), (h, w, tokyo)


def test_jitter_path_with_png_files_matches_host_train_transform(eng):
    from openibl_b200.utils.data import get_transformer_train
    from openibl_b200.utils.data.gpu_jpeg import decode_batch
    files = [png_file(image(480, 640, 2, 41), 2), png_file(image(480, 640, 0, 42), 0),
             png_file(image(300, 400, 3, 43), 3, palette=_pal(4)), _jpeg(image(480, 640, 2, 44), quality=92)]
    for h, w in ((480, 640), (240, 320)):
        host, dev = get_transformer_train(h, w), get_transformer_train(h, w, device_decode=True)
        want, carriers = [], []
        for i, f in enumerate(files):
            torch.manual_seed(70 + i)
            want.append(host(Image.open(io.BytesIO(f)).convert("RGB")))
            torch.manual_seed(70 + i)
            carriers.append(dev(f, f"p{i}.png"))
        got = decode_batch(carriers).cpu()
        for i in range(len(files)):
            assert torch.equal(got[i], want[i]), (h, w, i, (got[i] - want[i]).abs().max())


def _model():
    from openibl_b200 import models, synth
    torch.manual_seed(3)
    base = models.create("vgg16", pretrained=False)
    pool = models.create("netvlad", dim=base.feature_dim)
    p = synth.make_netvlad_params(seed=3, sharp=True)
    pool.centroids.data.copy_(p["centroids"])
    pool.conv.weight.data.copy_(p["conv_weight"])
    return models.create("embednet", base, pool).cuda()


@pytest.fixture(scope="module")
def tokyo(tmp_path_factory):
    """A Tokyo-shaped tree (meta.json / splits.json, JPEG queries, PNG database) made from the synthetic Pittsburgh
    splits, as the reference's Tokyo loader names its database files .png."""
    from openibl_b200 import datasets
    tmp = tmp_path_factory.mktemp("png_tokyo")
    proot = str(tmp / "pitts")
    datasets.write_synthetic_pitts_tree(proot, scale="30k")
    datasets.create("pitts", proot, scale="30k", verbose=False)
    root = str(tmp / "tokyo")
    shutil.copytree(os.path.join(proot, "raw"), os.path.join(root, "raw"))
    meta = json.load(open(os.path.join(proot, "meta_30k.json")))
    splits = json.load(open(os.path.join(proot, "splits_30k.json")))
    db = {pid for k in ("db_train", "db_val", "db_test") for pid in splits[k]}
    for pid in db:
        names = []
        for name in meta["identities"][pid]:
            src = os.path.join(root, "raw", name)
            dst = src[:-3] + "png"
            Image.open(src).convert("RGB").save(dst, "PNG")
            names.append(name[:-3] + "png")
        meta["identities"][pid] = names
    json.dump(meta, open(os.path.join(root, "meta.json"), "w"))
    json.dump(splits, open(os.path.join(root, "splits.json"), "w"))
    ds = datasets.create("tokyo", root, verbose=False)
    assert ds.db_test and all(it[0].endswith(".png") for it in ds.db_test)
    assert all(it[0].endswith(".jpg") for it in ds.q_test)
    return ds


def _loader(ds, items, device_decode, h=96, w=128):
    from torch.utils.data import DataLoader
    from openibl_b200.utils.data import Preprocessor, get_transformer_test
    pre = Preprocessor(items, root=ds.images_dir, transform=get_transformer_test(h, w, device_decode=device_decode))
    return DataLoader(pre, batch_size=8, num_workers=2, shuffle=False, pin_memory=True)


def test_tokyo_png_database_is_decoded_on_the_device(tokyo, monkeypatch):
    from openibl_b200.utils.data import gpu_jpeg
    files = [open(os.path.join(tokyo.images_dir, it[0]), "rb").read() for it in tokyo.db_test[:8]]

    def refuse(data):
        raise AssertionError("a PNG reached the host decoder")
    monkeypatch.setattr(gpu_jpeg, "_host_decode", refuse)
    gpu_jpeg.decode_to_tensor(files, 96, 128)


def test_tokyo_features_and_recalls_identical_with_device_decode(tokyo):
    from openibl_b200.evaluators import Evaluator, extract_features
    model = _model()
    items = sorted(list(set(tokyo.q_test) | set(tokyo.db_test)))
    host = extract_features(model, _loader(tokyo, items, False), items, print_freq=1000)
    dev = extract_features(model, _loader(tokyo, items, True), items, print_freq=1000)
    assert list(host) == list(dev)
    for k in host:
        assert torch.equal(host[k], dev[k]), k
    ev = Evaluator(model)
    rec = []
    for dd in (False, True):
        rec.append(ev.evaluate(_loader(tokyo, tokyo.q_test, dd), items, tokyo.q_test, tokyo.db_test, tokyo.test_pos,
                               gallery_loader=_loader(tokyo, tokyo.db_test, dd), vlad=True, nms=True))
    assert np.array_equal(np.asarray(rec[0]), np.asarray(rec[1])), rec


def test_decode_jpeg_names_corrupt_jpegs_and_pngs_together(eng):
    good = _jpeg(image(64, 80, 2, 61), quality=90)
    sos = good.index(b"\xff\xda")
    mid = (sos + len(good)) // 2
    bad_jpeg = good[:mid] + b"\xff\x00" * 8 + good[mid + 16:]          # 64 one-bits: no Huffman code
    a = image(6, 7, 2, 5)
    bad_png = corrupt_cases()["wrong Adler-32"][0]
    with pytest.raises(RuntimeError, match=r"JPEG entropy data in file\(s\) \[1\] and corrupt PNG image data in "
                                           r"file\(s\) \[2\]"):
        eng.decode_jpeg([good, bad_jpeg, bad_png, png_file(a, 2)])

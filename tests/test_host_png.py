"""PNG parse (csrc/png.cu, ibl_png_parse) and a Python model of the device decode, on the CPU.

`png_file` writes PNGs the tests need and Pillow's encoder does not: every filter type, any zlib level and strategy,
CINFO < 7, IDAT chunks of any size, and the corruptions of the acceptance table.  The model restates the kernels'
algorithms (canonical tables with a primary lookup, a ring-buffer inflate whose match bytes repeat byte i mod d, the
diagonal unfilter wavefront) and is checked against zlib and Pillow."""
import io
import struct
import zlib

import numpy as np
import pytest
from PIL import Image

SIG = b"\x89PNG\r\n\x1a\n"
BPP = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}


def chunk(cid: bytes, data: bytes, crc=None) -> bytes:
    c = zlib.crc32(cid + data) if crc is None else crc
    return struct.pack(">I", len(data)) + cid + data + struct.pack(">I", c & 0xFFFFFFFF)


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def filter_rows(px: np.ndarray, filters, bpp: int) -> bytes:
    """px uint8 [H, W*bpp] -> the filtered scanlines (filter byte + bytes), row r with filter filters[r % len]."""
    h, n = px.shape
    out = bytearray()
    prev = np.zeros(n, np.int32)
    for r in range(h):
        x = px[r].astype(np.int32)
        left = np.concatenate([np.zeros(bpp, np.int32), x[:-bpp]])
        ul = np.concatenate([np.zeros(bpp, np.int32), prev[:-bpp]])
        f = filters[r % len(filters)]
        pred = [0, left, prev, (left + prev) >> 1, _paeth(left, prev, ul) if f == 4 else 0][f]
        out.append(f)
        out += ((x - pred) & 255).astype(np.uint8).tobytes()
        prev = x
    return bytes(out)


def png_file(a: np.ndarray, ct: int, filters=(0, 1, 2, 3, 4), level=6, strategy=zlib.Z_DEFAULT_STRATEGY, wbits=15,
             split=None, palette=None, trns=None, pre=(), post=(), iend=True, zlib_stream=None, ihdr=None) -> bytes:
    """A PNG of `a` (uint8 [H, W, bpp] or [H, W]) with colour type ct, bit depth 8."""
    a = np.asarray(a, np.uint8)
    h, w = a.shape[:2]
    bpp = BPP[ct]
    raw = filter_rows(a.reshape(h, w * bpp), list(filters), bpp)
    if zlib_stream is None:
        co = zlib.compressobj(level, zlib.DEFLATED, wbits, 9, strategy)
        zlib_stream = co.compress(raw) + co.flush()
    f = SIG + chunk(b"IHDR", ihdr if ihdr is not None else struct.pack(">IIBBBBB", w, h, 8, ct, 0, 0, 0))
    for c in pre:
        f += c
    if palette is not None:
        f += chunk(b"PLTE", bytes(np.asarray(palette, np.uint8).reshape(-1)))
    if trns is not None:
        f += chunk(b"tRNS", trns)
    step = split or max(1, len(zlib_stream))
    for i in range(0, max(1, len(zlib_stream)), step):
        f += chunk(b"IDAT", zlib_stream[i: i + step])
    for c in post:
        f += c
    return f + (chunk(b"IEND", b"") if iend else b"")


def image(h, w, ct, seed, noise=False):
    r = np.random.default_rng(seed)
    bpp = BPP[ct]
    if noise:
        return r.integers(0, 256, (h, w, bpp), dtype=np.uint8)
    base = r.integers(0, 256, (h // 8 + 2, w // 8 + 2, bpp)).astype(np.float64)
    yy = np.linspace(0, base.shape[0] - 1.001, h)[:, None]
    xx = np.linspace(0, base.shape[1] - 1.001, w)[None, :]
    a = base[yy.astype(int), xx.astype(int)]
    a = np.clip(a + r.integers(-6, 7, a.shape), 0, 255).astype(np.uint8)
    if ct == 3:
        a = a % 200
    return a


def pillow(data):
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


def pillow_ok(data):
    try:
        pillow(data)
        return True
    except Exception:
        return False


def parse(data):
    from openibl_b200 import _cabi
    return _cabi.png_parse(data)


# ---- acceptance: which files the device takes, and why it leaves the others to Pillow --------------------------------

def _base(ct=2, h=6, w=7, **kw):
    pal = np.random.default_rng(1).integers(0, 256, (256, 3)) if ct == 3 else None
    return png_file(image(h, w, ct, 5), ct, palette=kw.pop("palette", pal), **kw)


def corrupt_cases():
    """name -> (file, Pillow decodes it, device decodes it: "ok" / "reject" / "error")."""
    good = _base()
    a = image(6, 7, 2, 5)
    raw = filter_rows(a.reshape(6, 21), [0, 1, 2, 3, 4], 3)
    z = zlib.compress(raw, 6)
    ihdr_at = good.index(b"IHDR")
    big = image(480, 640, 2, 9)
    zbig = zlib.compress(filter_rows(big.reshape(480, 1920), [0, 1, 2, 3, 4], 3), 6)
    bad_adler = lambda s: s[:-4] + bytes([s[-4] ^ 0x55]) + s[-3:]
    raw_bad_filter = bytearray(raw)
    raw_bad_filter[22] = 5
    co = zlib.compressobj(6)
    cut_final = co.compress(raw) + co.flush(zlib.Z_SYNC_FLUSH)       # rows complete, no final block, no Adler
    return {
        "bad IDAT CRC": (_idat_crc(png_file(a, 2, zlib_stream=z)), True, "ok"),
        "bad CRC before IDAT": (good[:ihdr_at + 17] + bytes([good[ihdr_at + 17] ^ 1]) + good[ihdr_at + 18:],
                                False, "reject"),
        "no IEND": (png_file(a, 2, zlib_stream=z, iend=False), True, "ok"),
        "no Adler-32": (png_file(a, 2, zlib_stream=z[:-4]), True, "ok"),
        "wrong Adler-32": (png_file(a, 2, zlib_stream=bad_adler(z)), False, "error"),
        "wrong Adler-32 480x640": (png_file(big, 2, zlib_stream=bad_adler(zbig)), False, "error"),
        "wrong Adler-32 480x640 8KiB IDATs": (png_file(big, 2, zlib_stream=bad_adler(zbig), split=8192), False,
                                              "error"),
        "junk after the stream": (png_file(a, 2, zlib_stream=z + b"junkjunk"), True, "ok"),
        "more rows than the image": (png_file(a, 2, zlib_stream=zlib.compress(raw + raw[:44], 6)), True, "ok"),
        "stream ends before the last row": (png_file(a, 2, zlib_stream=zlib.compress(raw[:-5], 6)), False, "error"),
        "stream cut before the last row": (png_file(a, 2, zlib_stream=z[: len(z) // 2]), False, "error"),
        "filter type 5": (png_file(a, 2, zlib_stream=zlib.compress(bytes(raw_bad_filter), 6)), False, "error"),
        "cut after the last row, before the final block": (png_file(a, 2, zlib_stream=cut_final), True, "ok"),
    }


def _idat_crc(f):
    i = f.index(b"IDAT")
    n = struct.unpack(">I", f[i - 4: i])[0]
    j = i + 4 + n
    return f[:j] + bytes([f[j] ^ 0xFF]) + f[j + 1:]


def test_corrupt_cases_match_the_acceptance_table():
    for name, (f, pil, dev) in corrupt_cases().items():
        assert pillow_ok(f) == pil, name
        p = parse(f)
        assert p["ok"] == (dev != "reject"), (name, p["reason"])


def _reject_cases():
    a1 = image(5, 6, 0, 3)
    return {
        "bit depth is not 8": [png_file(a1, 0, ihdr=struct.pack(">IIBBBBB", 6, 5, d, 0, 0, 0, 0)) for d in (1, 2, 4, 16)],
        "interlaced": [png_file(a1, 0, ihdr=struct.pack(">IIBBBBB", 6, 5, 8, 0, 0, 0, 1))],
        "APNG": [png_file(a1, 0, pre=[chunk(b"acTL", struct.pack(">II", 1, 0))])],
        "zlib preset dictionary": [png_file(a1, 0, zlib_stream=b"\x78\xbb" + b"\0" * 12)],
        "palette image without PLTE": [png_file(image(5, 6, 3, 3), 3, palette=None)],
        "zero width or height": [png_file(np.zeros((1, 1, 1), np.uint8), 0,
                                          ihdr=struct.pack(">IIBBBBB", w, h, 8, 0, 0, 0, 0)) for w, h in ((0, 1), (1, 0))],
        "bad CRC before IDAT": [png_file(a1, 0, pre=[chunk(b"tEXt", b"a\0b", crc=1)])],
        "zlib window larger than 32 KiB": [png_file(a1, 0, zlib_stream=b"\x88\x1c" + b"\0" * 8)],
    }


@pytest.mark.parametrize("reason", list(_reject_cases()))
def test_parse_rejects_what_pillow_keeps(reason):
    for f in _reject_cases()[reason]:
        p = parse(f)
        assert not p["ok"] and p["reason"] == reason, (reason, p["reason"])


@pytest.mark.parametrize("ct", [0, 2, 3, 4, 6])
def test_parse_accepts_every_colour_type(ct):
    f = _base(ct, 9, 11, trns=b"\x00\x10" if ct == 0 else None)
    p = parse(f)
    assert p["ok"], p["reason"]
    assert (p["width"], p["height"], p["color_type"], p["bit_depth"]) == (11, 9, ct, 8)
    assert p["palette_size"] == (256 if ct == 3 else 0)
    assert p["zlib_bytes"] > 2


def test_parse_accepts_what_pillow_writes():
    for mode in ("L", "RGB", "RGBA", "LA", "P"):
        im = Image.fromarray(image(33, 47, 2, 7)).convert(mode)
        b = io.BytesIO()
        im.save(b, "PNG")
        assert parse(b.getvalue())["ok"], mode


def test_short_palette_reads_black_past_its_end_in_pillow():
    a = np.full((2, 3, 1), 7, np.uint8)
    a[0, 0] = 1
    f = png_file(a, 3, palette=[[10, 20, 30], [40, 50, 60]])
    assert parse(f)["ok"] and parse(f)["palette_size"] == 2
    want = pillow(f)
    assert want[0, 0].tolist() == [40, 50, 60] and want[1, 1].tolist() == [0, 0, 0]


# ---- a Python model of the device algorithm ----------------------------------------------------------------------

LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227,
         258]
LEXT = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
         6145, 8193, 12289, 16385, 24577]
DEXT = [max(0, i // 2 - 1) for i in range(30)]
CLORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


class Corrupt(Exception):
    pass


class Code:
    """build_code: primary table of `root` bits (sym, len) plus canonical count/sorted for longer codes."""

    def __init__(self, lens, root):
        self.root = root
        self.count = [0] * 16
        for l in lens:
            self.count[l] += 1
        self.count[0] = 0
        left, maxl = 1, 0
        for l in range(1, 16):
            left = (left << 1) - self.count[l]
            if left < 0:
                break
            if self.count[l]:
                maxl = l
        self.kind = -1 if left < 0 else 0 if left == 0 else (2 if maxl == 0 else 3 if maxl == 1 else 1)
        self.tab = [None] * (1 << root)
        self.sorted = []
        if self.kind < 0:
            return
        nxt, code = [0] * 16, 0
        for l in range(1, 16):
            code = (code + (self.count[l - 1] if l > 1 else 0)) << 1
            nxt[l] = code
        self.sorted = [s for l in range(1, 16) for s, m in enumerate(lens) if m == l]
        for s, l in enumerate(lens):
            if l:
                c = nxt[l]
                nxt[l] += 1
                if l <= root:
                    rev = int(format(c, f"0{l}b")[::-1], 2)
                    for e in range(rev, 1 << root, 1 << l):
                        self.tab[e] = (s, l)

    def decode(self, br):
        e = self.tab[br.peek(self.root)]
        if e:
            br.drop(e[1])
            return e[0]
        code = first = index = 0
        bits = br.peek(15)
        for l in range(1, 16):
            code |= (bits >> (l - 1)) & 1
            cnt = self.count[l]
            if code - cnt < first:
                br.drop(l)
                return self.sorted[index + code - first]
            index += cnt
            first = (first + cnt) << 1
            code <<= 1
        return -1


class Bits:
    def __init__(self, data):
        self.data, self.pos = data, 16               # past the zlib header

    def peek(self, n):
        v = 0
        for k in range(n):
            i = self.pos + k
            if i < len(self.data) * 8:
                v |= ((self.data[i >> 3] >> (i & 7)) & 1) << k
        return v

    def drop(self, n):
        self.pos += n

    def take(self, n):
        v = self.peek(n)
        self.drop(n)
        return v

    def over(self):
        return self.pos > len(self.data) * 8


def model_inflate(z: bytes):
    """png_inflate_kernel on one stream: (output bytes, state) with state 1 final block, 2 input ran out, 3 corrupt.
    Matches go through a 64 KiB ring exactly as the kernel's lanes copy them."""
    br = Bits(z)
    ring = bytearray(65536)
    out = bytearray()
    P = 0

    def emit(b):
        nonlocal P
        ring[P & 65535] = b
        out.append(b)
        P += 1

    while True:
        hdr = br.take(3)
        if br.over():
            return out, 2
        t = hdr >> 1
        if t == 0:
            br.drop(-br.pos & 7)
            ln, nl = br.take(16), br.take(16)
            if br.over():
                return out, 2
            if ln ^ 0xFFFF != nl:
                return out, 3
            bp = br.pos >> 3
            n = min(ln, len(z) - bp)
            for b in z[bp: bp + n]:
                emit(b)
            br.pos = (bp + n) * 8
            if n < ln:
                return out, 2
        elif t == 3:
            return out, 3
        else:
            if t == 1:
                lens = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8 + [5] * 30
                hlit = 288
            else:
                hlit, hdist, hclen = br.take(5) + 257, br.take(5) + 1, br.take(4) + 4
                if br.over():
                    return out, 2
                if hlit > 286 or hdist > 30:
                    return out, 3
                cll = [0] * 19
                for k in range(hclen):
                    cll[CLORDER[k]] = br.take(3)
                if br.over():
                    return out, 2
                cl = Code(cll, 7)
                if cl.kind != 0:
                    return out, 3
                lens = []
                while len(lens) < hlit + hdist:
                    sym = cl.decode(br)
                    rep, val = 1, sym
                    if sym == 16:
                        if not lens:
                            return out, (2 if br.over() else 3)
                        rep, val = 3 + br.take(2), lens[-1]
                    elif sym == 17:
                        rep, val = 3 + br.take(3), 0
                    elif sym == 18:
                        rep, val = 11 + br.take(7), 0
                    if br.over():
                        return out, 2
                    if len(lens) + rep > hlit + hdist:
                        return out, 3
                    lens += [val] * rep
                if lens[256] == 0:
                    return out, 3
            lit, dist = Code(lens[:hlit], 10), Code(lens[hlit:], 8)
            if t == 2 and (lit.kind in (-1, 1) or dist.kind in (-1, 1)):
                return out, 3
            while True:
                sym = lit.decode(br)
                if sym < 0 or sym >= 286:
                    return out, (2 if br.pos + 15 > len(z) * 8 else 3)
                if sym < 256:
                    if br.over():
                        return out, 2
                    emit(sym)
                elif sym == 256:
                    if br.over():
                        return out, 2
                    break
                else:
                    ln = LBASE[sym - 257] + br.take(LEXT[sym - 257])
                    ds = dist.decode(br)
                    if ds < 0 or ds >= 30:
                        return out, (2 if br.pos + 15 > len(z) * 8 else 3)
                    d = DBASE[ds] + br.take(DEXT[ds])
                    if br.over():
                        return out, 2
                    if d > P:
                        return out, 3
                    src = [ring[(P - d + (i if i < d else i % d)) & 65535] for i in range(ln)]
                    for b in src:
                        emit(b)
        if hdr & 1:
            return out, 1


def model_unfilter(rows: bytes, h: int, w: int, bpp: int, band=4):
    """png_unfilter_kernel: thread r of a band reconstructs pixel t - r at step t; pixel above from the step before."""
    rb = 1 + w * bpp
    ws = bytearray(rows)
    out = np.zeros((h, w * bpp), np.uint8)
    for r0 in range(0, h, band):
        rows_n = min(band, h - r0)
        up_px = [[None] * band, [None] * band]
        left = [bytes(bpp)] * band
        upleft = [bytes(bpp)] * band
        for t in range(w + rows_n - 1):
            for tid in range(rows_n):
                x, r = t - tid, r0 + tid
                if not 0 <= x < w:
                    continue
                if tid > 0:
                    up = up_px[(t - 1) & 1][tid - 1]
                elif r > 0:
                    up = bytes(ws[(r - 1) * rb + 1 + x * bpp: (r - 1) * rb + 1 + (x + 1) * bpp])
                else:
                    up = bytes(bpp)
                ft = ws[r * rb]
                assert ft <= 4
                px = bytearray(bpp)
                for k in range(bpp):
                    a, b, c = left[tid][k], up[k], upleft[tid][k]
                    v = ws[r * rb + 1 + x * bpp + k]
                    v += [0, a, b, (a + b) >> 1, int(_paeth(np.int32(a), np.int32(b), np.int32(c)))][ft]
                    px[k] = v & 255
                up_px[t & 1][tid] = bytes(px)
                if tid == rows_n - 1:
                    ws[r * rb + 1 + x * bpp: r * rb + 1 + (x + 1) * bpp] = px
                left[tid], upleft[tid] = bytes(px), up
                out[r, x * bpp: (x + 1) * bpp] = list(px)
    return out


STRATEGIES = [(0, zlib.Z_DEFAULT_STRATEGY), (1, zlib.Z_DEFAULT_STRATEGY), (6, zlib.Z_DEFAULT_STRATEGY),
              (9, zlib.Z_DEFAULT_STRATEGY), (6, zlib.Z_FIXED), (6, zlib.Z_HUFFMAN_ONLY), (6, zlib.Z_RLE)]


@pytest.mark.parametrize("level,strategy", STRATEGIES)
def test_model_inflate_matches_zlib(level, strategy):
    r = np.random.default_rng(level * 10 + strategy)
    data = bytes(r.integers(0, 4, 3000, dtype=np.uint8)) + bytes(700) + bytes(r.integers(0, 256, 900, dtype=np.uint8))
    co = zlib.compressobj(level, zlib.DEFLATED, 15, 9, strategy)
    z = co.compress(data) + co.flush()
    out, state = model_inflate(z)
    assert state == 1 and bytes(out) == zlib.decompress(z) == data


def test_model_inflate_long_matches_and_small_window():
    # 258-byte matches at distance 32768 (the window's far end), and d < len runs
    block = bytes(np.random.default_rng(3).integers(0, 256, 32768, dtype=np.uint8))
    data = block + block[:2000] + b"ab" * 600
    z = zlib.compress(data, 9)
    out, state = model_inflate(z)
    assert state == 1 and bytes(out) == data
    # CINFO < 7: the encoder keeps its distances inside 512 bytes, the header says so, the decode does not care
    co = zlib.compressobj(9, zlib.DEFLATED, 9)
    z9 = co.compress(data) + co.flush()
    assert z9[0] >> 4 == 1
    out, state = model_inflate(z9)
    assert state == 1 and bytes(out) == data


def test_model_inflate_flags_corrupt_streams():
    data = bytes(np.random.default_rng(4).integers(0, 8, 5000, dtype=np.uint8))
    z = zlib.compress(data, 6)
    assert model_inflate(z[:len(z) // 2])[1] == 2                      # input runs out
    assert model_inflate(b"\x78\x9c" + bytes([0b111]))[1] == 3          # block type 3
    assert model_inflate(b"\x78\x9c\x01\x05\x00\x00\x00")[1] == 3      # stored LEN/NLEN mismatch
    # a distance past the first byte: fixed block, literal 'a', then length 3 distance 2
    assert model_inflate(_fixed_stream([("lit", 97), ("match", 3, 2)]))[1] == 3
    assert model_inflate(_fixed_stream([("lit", 97), ("match", 3, 1)]))[0] == b"aaaa"


def _fixed_stream(tokens):
    """A one-block fixed-Huffman stream (no Adler) from literal / (length 3..10, distance 1..4) tokens."""
    bits = [1, 1, 0]                                                     # BFINAL, BTYPE=01 (LSB first)

    def code(v, n):                                                      # Huffman codes go MSB first
        bits.extend((v >> (n - 1 - k)) & 1 for k in range(n))
    for t in tokens:
        if t[0] == "lit":
            code(0x30 + t[1], 8) if t[1] < 144 else code(0x190 + t[1] - 144, 9)
        else:
            code(t[1] - 3 + 1, 7)                                        # length codes 257..264: 7-bit 1..8
            code(t[2] - 1, 5)                                            # distance codes 0..3, no extra bits
    code(0, 7)                                                           # end of block
    bits += [0] * (-len(bits) % 8)
    return b"\x78\x9c" + bytes(sum(b << k for k, b in enumerate(bits[i: i + 8])) for i in range(0, len(bits), 8))


@pytest.mark.parametrize("ct", [0, 2, 3, 4, 6])
def test_model_decode_matches_pillow(ct):
    a = image(11, 13, ct, 20 + ct)
    pal = np.random.default_rng(2).integers(0, 256, (256, 3)) if ct == 3 else None
    f = png_file(a, ct, palette=pal, level=9)
    bpp = BPP[ct]
    i = f.index(b"IDAT")
    n = struct.unpack(">I", f[i - 4: i])[0]
    rows, state = model_inflate(f[i + 4: i + 4 + n])
    assert state == 1
    px = model_unfilter(bytes(rows[: 11 * (1 + 13 * bpp)]), 11, 13, bpp).reshape(11, 13, bpp)
    if ct == 3:
        rgb = np.asarray(pal, np.uint8)[px[..., 0]]
    elif ct in (0, 4):
        rgb = np.repeat(px[..., :1], 3, axis=2)
    else:
        rgb = px[..., :3]
    assert np.array_equal(rgb, pillow(f))


# ---- hand-built dynamic blocks: zlib's (inftrees.c) rules for which code sets are valid ---------------------------

def _canon(lens):
    """symbol -> (code, length) of the canonical code with these lengths (DEFLATE 3.2.2)."""
    count = [0] * 16
    for l in lens:
        count[l] += 1
    count[0] = 0
    nxt, code = [0] * 16, 0
    for l in range(1, 16):
        code = (code + count[l - 1]) << 1
        nxt[l] = code
    out = {}
    for s, l in enumerate(lens):
        if l:
            out[s] = (nxt[l], l)
            nxt[l] += 1
    return out


class _BitWriter:
    def __init__(self):
        self.bits = []

    def lsb(self, v, n):
        self.bits += [(v >> k) & 1 for k in range(n)]

    def huff(self, code):
        c, n = code
        self.bits += [(c >> (n - 1 - k)) & 1 for k in range(n)]

    def align(self):
        self.bits += [0] * (-len(self.bits) % 8)

    def tobytes(self):
        self.align()
        return bytes(sum(b << k for k, b in enumerate(self.bits[i: i + 8])) for i in range(0, len(self.bits), 8))


def dynamic_stream(lit_lens, dist_lens, tokens, stored_prefix=b"", cmf=0x78):
    """A zlib stream: an optional non-final stored block holding `stored_prefix`, then one final dynamic block with
    the given literal/length and distance code lengths (any, valid or not) and tokens: ints are literals or 256,
    (length 3..10, distance code) pairs are matches.  The Adler-32 covers what a valid decode produces."""
    bw = _BitWriter()
    out = bytearray(stored_prefix)
    if stored_prefix:
        bw.lsb(0, 3)
        bw.align()
        bw.lsb(len(stored_prefix), 16)
        bw.lsb(len(stored_prefix) ^ 0xFFFF, 16)
        for b in stored_prefix:
            bw.lsb(b, 8)
    lit_lens = list(lit_lens) + [0] * (257 - len(lit_lens))
    bw.lsb(1, 1)
    bw.lsb(2, 2)
    bw.lsb(len(lit_lens) - 257, 5)
    bw.lsb(len(dist_lens) - 1, 5)
    bw.lsb(19 - 4, 4)
    cl_lens = [4] * 13 + [5] * 6                     # a complete code-length code over symbols 0..18
    for k in range(19):
        bw.lsb(cl_lens[CLORDER[k]], 3)
    cl = _canon(cl_lens)
    for l in lit_lens + list(dist_lens):
        bw.huff(cl[l])
    lit, dist = _canon(lit_lens), _canon(dist_lens)
    for t in tokens:
        if isinstance(t, tuple):
            ln, dc = t
            bw.huff(lit[254 + ln])                   # length codes 257..264 are lengths 3..10, no extra bits
            bw.huff(dist[dc])
            d = DBASE[dc]
            for _ in range(ln):
                out.append(out[-d] if d <= len(out) else 0)
        else:
            bw.huff(lit[t])
            if t < 256:
                out.append(t)
    hdr = bytes([cmf, (31 - (cmf * 256) % 31) % 31])
    return hdr + bw.tobytes() + struct.pack(">I", zlib.adler32(bytes(out))), bytes(out)


def _lits(*pairs, n=258):
    lens = [0] * n
    for s, l in pairs:
        lens[s] = l
    return lens


ROW = bytes([0, 97, 97, 97, 97])                     # one 4-pixel grey row, filter None


def huffman_cases():
    """name -> (zlib stream, zlib and the device accept it).  Invalid code sets follow a stored block that already
    holds the whole image, and the bad block holds nothing but its end code, so only the table check can reject it."""
    ok_lit = _lits((0, 2), (97, 2), (256, 2), (257, 2))
    return {
        "single one-bit distance code": (dynamic_stream(ok_lit, [1], [0, 97, (3, 0), 256])[0], True),
        "no distance codes, literals only": (dynamic_stream(ok_lit, [0], [0, 97, 97, 97, 97, 256])[0], True),
        "single one-bit literal/length code": (dynamic_stream(_lits((256, 1)), [1], [256], ROW)[0], True),
        "over-subscribed literal/length code": (
            dynamic_stream(_lits((0, 1), (97, 1), (256, 1)), [1], [256], ROW)[0], False),
        "incomplete literal/length code": (dynamic_stream(_lits((0, 2), (97, 2), (256, 2)), [1], [256], ROW)[0], False),
        "incomplete two-bit distance code": (dynamic_stream(ok_lit, [2, 2], [256], ROW)[0], False),
        "over-subscribed distance code": (dynamic_stream(ok_lit, [1, 1, 1], [256], ROW)[0], False),
        "distance past the output": (dynamic_stream(ok_lit, [1, 1], [0, (3, 1), 97, 256])[0], False),
        "no end-of-block code": (dynamic_stream(_lits((0, 1), (97, 1), n=257), [1], [], ROW)[0], False),
    }


def _zlib_ok(z):
    try:
        zlib.decompress(z)
        return True
    except zlib.error:
        return False


@pytest.mark.parametrize("name", list(huffman_cases()))
def test_model_follows_zlib_on_code_sets(name):
    z, ok = huffman_cases()[name]
    assert _zlib_ok(z) == ok, name
    out, state = model_inflate(z)
    if ok:
        assert state == 1 and bytes(out) == zlib.decompress(z) == ROW
    else:
        assert state == 3, state
    assert pillow_ok(png_file(np.zeros((1, 4, 1), np.uint8), 0, zlib_stream=z)) == ok


def far_match_cinfo1():
    """A wbits=15 stream whose matches reach 32 KiB back, with its header rewritten to CINFO = 1 (a 512-byte
    window): non-strict zlib, and so Pillow, still decodes it."""
    base = np.random.default_rng(5).integers(0, 256, (32, 1024, 1), dtype=np.uint8)
    a = np.concatenate([base, base])
    raw = filter_rows(a.reshape(64, 1024), [0], 1)
    z = zlib.compress(raw, 9)
    cmf = 0x18
    flg = (z[1] & 0xE0) | ((31 - ((cmf << 8) | (z[1] & 0xE0)) % 31) % 31)
    return a, bytes([cmf, flg]) + z[2:]


def test_model_and_pillow_take_cinfo_below_7_with_far_matches():
    a, z = far_match_cinfo1()
    assert z[0] >> 4 == 1 and ((z[0] << 8) | z[1]) % 31 == 0
    f = png_file(a, 0, zlib_stream=z)
    assert parse(f)["ok"]
    assert np.array_equal(pillow(f)[..., 0], a[..., 0])
    out, state = model_inflate(z)
    assert state == 1 and bytes(out) == zlib.decompress(z)


def test_parse_rejects_chrm_pillow_cannot_unpack():
    a = image(5, 6, 2, 3)
    bad = png_file(a, 2, pre=[chunk(b"cHRM", b"\0" * 30)])
    assert not pillow_ok(bad)
    assert parse(bad)["reason"] == "cHRM length not a multiple of 4"
    good = png_file(a, 2, pre=[chunk(b"cHRM", b"\0" * 32)])
    assert pillow_ok(good) and parse(good)["ok"]

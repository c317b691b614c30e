"""Host side of the device JPEG decoder (csrc/jpeg.cu), no GPU: the parser against Pillow's own reading of the same
bytes, its rejections, and a Python model of the parallel entropy decode (self-synchronising runs, fix-up passes,
block scan, writing pass) against the sequential decode."""
import io
import random

import numpy as np
import pytest
from PIL import Image

from openibl_b200 import _cabi


def _img(h, w, seed, mode="RGB"):
    r = np.random.default_rng(seed)
    base = r.integers(0, 256, (h // 8 + 2, w // 8 + 2, 3)).astype(np.uint8)
    a = np.asarray(Image.fromarray(base).resize((w, h), Image.BILINEAR)).astype(np.int16)
    a = np.clip(a + r.integers(-20, 21, a.shape), 0, 255).astype(np.uint8)
    im = Image.fromarray(a)
    return im.convert("L") if mode == "L" else im


def _jpeg(im, **kw):
    b = io.BytesIO()
    im.save(b, "JPEG", **kw)
    return b.getvalue()


SAMPLING = {0: (1, 1), 1: (2, 1), 2: (2, 2)}


@pytest.mark.parametrize("sub", [0, 1, 2])
@pytest.mark.parametrize("quality", [50, 92, 100])
@pytest.mark.parametrize("extra", [{}, {"optimize": True}, {"restart_marker_blocks": 3}, {"restart_marker_rows": 1},
                                   {"exif": b"Exif\x00\x00" + b"II*\x00\x08\x00\x00\x00\x00\x00"}])
def test_parse_matches_pillow(sub, quality, extra):
    data = _jpeg(_img(37, 53, quality + sub), quality=quality, subsampling=sub, **extra)
    info = _cabi.jpeg_parse(data)
    ref = Image.open(io.BytesIO(data))
    assert info["ok"], info["reason"]
    assert (info["width"], info["height"]) == ref.size and ref.mode == "RGB" and info["components"] == 3
    assert (info["h_samp"], info["v_samp"]) == SAMPLING[sub]
    hs, vs = SAMPLING[sub]
    assert info["mcus"] == -(-37 // (8 * vs)) * -(-53 // (8 * hs))
    if "restart_marker_blocks" in extra or "restart_marker_rows" in extra:
        assert info["restart_interval"] > 0
        assert info["intervals"] == -(-info["mcus"] // info["restart_interval"])
    else:
        assert info["intervals"] == 1
    # destuffed entropy bytes: the scan's bytes minus one per stuffed 0x00 and two per RSTn
    assert 0 < info["entropy_bytes"] < len(data)


@pytest.mark.parametrize("size", [(1, 1), (7, 9), (4000, 3)])
def test_parse_grayscale_and_extreme_sizes(size):
    h, w = size
    for mode in ("L", "RGB"):
        data = _jpeg(_img(h, w, 1, mode), quality=90)
        info = _cabi.jpeg_parse(data)
        ref = Image.open(io.BytesIO(data))
        assert info["ok"], info["reason"]
        assert (info["width"], info["height"]) == ref.size
        assert info["components"] == (1 if ref.mode == "L" else 3)


def _patch(data, marker, offset, value):
    """Set byte `offset` of the first segment with `marker` (offset 0 = first byte after the length field)."""
    i = data.index(bytes([0xFF, marker]))
    b = bytearray(data)
    b[i + 4 + offset] = value
    return bytes(b)


def test_parser_rejects_unsupported_kinds_with_reasons():
    im = _img(40, 48, 7)
    base = _jpeg(im, quality=80)
    cases = {
        "progressive": _jpeg(im, quality=80, progressive=True),
        "CMYK": _jpeg(im.convert("CMYK"), quality=80),
        "12-bit": _patch(base, 0xC0, 0, 12),
        "arithmetic": base.replace(b"\xff\xc0", b"\xff\xc9", 1),
        "sampling": _patch(base, 0xC0, 7, 0x12),           # luma 1x2 (4:4:0)
        "truncated": base[: len(base) // 2],
        "missing EOI": base[:-2],
        "bad segment length": base.replace(b"\xff\xdb\x00\x43", b"\xff\xdb\x00\x44", 1),
        "RGB-coded": _jpeg(im, quality=80, keep_rgb=True),
    }
    for want, data in cases.items():
        info = _cabi.jpeg_parse(data)
        assert not info["ok"] and info["status"] == 6, (want, info)
        assert want.lower().split()[0] in info["reason"].lower() or \
            (want == "sampling" and "sampling" in info["reason"]) or \
            (want == "CMYK" and "cmyk" in info["reason"].lower()), (want, info["reason"])
    assert "missing eoi" in _cabi.jpeg_parse(base[:-2])["reason"].lower()
    assert not _cabi.jpeg_parse(b"")["ok"] and not _cabi.jpeg_parse(b"\x89PNG\r\n\x1a\n")["ok"]


# ---- Python model of the parallel entropy decode ------------------------------------------------------------------
# Mirrors csrc/jpeg.cu: decode_run (one codeword at a time: DC difference, AC run/size, ZRL, EOB, block end past
# index 63), jpeg_sync_kernel (every run starts at "coefficient 0 of the MCU's first block" at its first bit, the
# first run of an interval in its known state), jpeg_fix_kernel (Jacobi passes: a run is decoded again from its
# predecessor's end state while any end state changes; invalid codes end a run in the invalid state), the exclusive
# scan of completed blocks, and jpeg_write_kernel (writes only blocks below the interval's block count).

INVALID = None


def canonical(lengths):
    """symbol -> code length  =>  {(length, code): symbol}, codes assigned as JPEG's canonical Huffman does."""
    code, out, prev = 0, {}, None
    for sym, ln in sorted(lengths.items(), key=lambda kv: (kv[1], kv[0])):
        if prev is not None:
            code = (code + 1) << (ln - prev)
        out[(ln, code)] = sym
        prev = ln
    return out


class Tables:
    def __init__(self, dc, ac):
        self.dc, self.ac = canonical(dc), canonical(ac)
        self.enc_dc = {s: (l, c) for (l, c), s in self.dc.items()}
        self.enc_ac = {s: (l, c) for (l, c), s in self.ac.items()}


def bit(bits, p):
    return bits[p] if p < len(bits) else 0          # the device pads every interval with zero bytes


def huff(table, bits, p):
    code = 0
    for ln in range(1, 17):
        code = (code << 1) | bit(bits, p + ln - 1)
        if (ln, code) in table:
            return table[(ln, code)], ln
    return None, 0


def take(bits, p, s):
    v = 0
    for i in range(s):
        v = (v << 1) | bit(bits, p + i)
    return v


def extend(v, s):
    return v - (1 << s) + 1 if v < (1 << (s - 1)) else v


def decode_run(bits, stop, tabs, bpm, state, emit=None):
    pos, blk, zz = state
    done = 0
    while pos < stop:
        t = tabs[blk]
        if zz == 0:
            s, ln = huff(t.dc, bits, pos)
            if s is None:
                return INVALID, done
            if emit:
                emit(done, 0, extend(take(bits, pos + ln, s), s) if s else 0)
            pos += ln + s
            zz = 1
        else:
            rs, ln = huff(t.ac, bits, pos)
            if rs is None:
                return INVALID, done
            r, s = rs >> 4, rs & 15
            if s:
                zz += r
                if emit:
                    emit(done, zz, extend(take(bits, pos + ln, s), s))
                zz += 1
                pos += ln + s
            else:
                zz = zz + 16 if r == 15 else 64
                pos += ln
        if zz >= 64:
            zz, blk = 0, (blk + 1) % bpm
            done += 1
    return (pos, blk, zz), done


def sequential(intervals, tabs, bpm):
    out = []
    for bits, nblocks in intervals:
        coef = [[0] * 64 for _ in range(nblocks)]

        def emit(k, zz, v):
            if k < nblocks:
                coef[k][min(zz, 63)] = v
        _, done = decode_run(bits, len(bits), tabs, bpm, (0, 0, 0), emit)
        assert done >= nblocks                                # past the last block only padding remains
        out.append(coef)
    return out


def parallel(intervals, tabs, bpm, run_bits):
    out, passes = [], 0
    for bits, nblocks in intervals:
        n = max(1, -(-len(bits) // run_bits))
        stop = [min((j + 1) * run_bits, len(bits)) for j in range(n)]
        # sync pass
        end, cnt = [], []
        for j in range(n):
            st, d = decode_run(bits, stop[j], tabs, bpm, (j * run_bits, 0, 0))
            end.append(st)
            cnt.append(d)

        def start(j):
            if j == 0:
                return (0, 0, 0)
            return end[j - 1] if end[j - 1] is not INVALID else (j * run_bits, 0, 0)
        need = [j != 0 for j in range(n)]
        while True:
            passes += 1
            new = {j: decode_run(bits, stop[j], tabs, bpm, start(j)) for j in range(n) if need[j]}
            chg = [False] * n
            for j, (st, d) in new.items():
                cnt[j] = d
                if st != end[j]:
                    end[j], chg[j] = st, True
            if not any(chg):
                break
            need = [j != 0 and chg[j - 1] for j in range(n)]
        first = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(int)
        coef = [[0] * 64 for _ in range(nblocks)]
        for j in range(n):
            assert j == 0 or end[j - 1] is not INVALID or first[j] >= nblocks

            def emit(k, zz, v, f=first[j]):
                if f + k < nblocks:
                    coef[f + k][min(zz, 63)] = v
            if j == 0 or end[j - 1] is not INVALID:
                decode_run(bits, stop[j], tabs, bpm, start(j), emit)
        out.append(coef)
    return out, passes


def encode(blocks, tabs_of, rng):
    """blocks: list of (block index in MCU, {zz: value}) -> bit list, padded with 1s to a byte as JPEG does."""
    bits = []

    def put(code_len, code):
        bits.extend((code >> (code_len - 1 - i)) & 1 for i in range(code_len))

    def put_value(v):
        s = 0 if v == 0 else int(abs(v)).bit_length()
        raw = v if v > 0 else v + (1 << s) - 1
        return s, raw
    for blk, coefs in blocks:
        t = tabs_of[blk]
        s, raw = put_value(coefs.get(0, 0))
        put(*t.enc_dc[s])
        put(s, raw) if s else None
        zz, last = 1, max([k for k in coefs if k > 0] or [0])
        while zz <= last:
            r = 0
            while coefs.get(zz, 0) == 0:
                r += 1
                zz += 1
                if r == 16:
                    put(*t.enc_ac[0xF0])
                    r = 0
            s, raw = put_value(coefs[zz])
            put(*t.enc_ac[(r << 4) | s])
            put(s, raw)
            zz += 1
        if zz < 64:
            put(*t.enc_ac[0x00])
    while len(bits) % 8:
        bits.append(1)
    return bits


def _random_blocks(rng, n, bpm, max_s, density):
    blocks = []
    for k in range(n):
        coefs = {0: rng.randint(-(1 << max_s) + 1, (1 << max_s) - 1)}
        for zz in range(1, 64):
            if rng.random() < density:
                v = 0
                while v == 0:
                    v = rng.randint(-(1 << max_s) + 1, (1 << max_s) - 1)
                coefs[zz] = v
        blocks.append((k % bpm, coefs))
    return blocks


def _full_tables(seed):
    """Skewed code lengths (1..16 bits) over every DC size and every AC run/size symbol."""
    rng = random.Random(seed)
    dc_syms = list(range(12))
    ac_syms = [0x00, 0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 11)]
    dc = {s: ln for s, ln in zip(dc_syms, [2, 3, 3, 3, 3, 3, 4, 5, 6, 7, 8, 9])}
    lens = [3] * 4 + [5] * 6 + [7] * 10 + [10] * 10 + [16] * 132
    rng.shuffle(ac_syms)
    ac = dict(zip(ac_syms, lens))
    return Tables(dc, ac)


def _kraft_ok(t):
    return sum(2.0 ** -ln for (ln, _c) in t.ac) <= 1 and sum(2.0 ** -ln for (ln, _c) in t.dc) <= 1


@pytest.mark.parametrize("run_bits", [32, 33, 57, 64, 256, 1024])
def test_sync_model_reproduces_sequential_decode(run_bits):
    rng = random.Random(run_bits)
    luma, chroma = _full_tables(1), _full_tables(2)
    assert _kraft_ok(luma) and _kraft_ok(chroma)
    bpm = 6                                                   # 4:2:0 MCU: four luma blocks, Cb, Cr
    tabs = [luma] * 4 + [chroma] * 2
    intervals = []
    for nmcu in (1, 3, 7, 20):                                # restart intervals of different lengths
        blocks = _random_blocks(rng, nmcu * bpm, bpm, max_s=8, density=0.15)
        intervals.append((encode(blocks, tabs, rng), nmcu * bpm))
    want = sequential(intervals, tabs, bpm)
    got, passes = parallel(intervals, tabs, bpm, run_bits)
    assert got == want


def test_sync_model_when_runs_never_synchronise():
    """Every codeword and every value field has an even length: a run started at an odd bit stays off the true
    boundaries forever, so every run's first guess is wrong and correctness rests on propagation alone."""
    dc = Tables({0: 2, 2: 2, 4: 2}, {0x00: 2, 0x02: 2, 0x12: 2})
    bpm = 1
    rng = random.Random(5)
    blocks = []
    for k in range(40):
        coefs = {0: rng.choice([0, 2, -2, 3, -3, 9, -9])}
        zz = 1
        while zz < 63 and rng.random() < 0.7:
            zz += rng.choice([0, 1])
            if zz < 64:
                coefs[zz] = rng.choice([2, -2, 3, -3])
            zz += 1
        blocks.append((0, coefs))
    bits = encode(blocks, [dc], rng)
    intervals = [(bits, 40)]
    want = sequential(intervals, [dc], bpm)
    for run_bits in (33, 35, 63):                             # odd run lengths: every other run starts at an odd bit
        n = -(-len(bits) // run_bits)
        odd = [j for j in range(1, n) if (j * run_bits) % 2]
        # from an odd start no codeword boundary of the run is a true one
        for j in odd:
            st, _ = decode_run(bits, min((j + 1) * run_bits, len(bits)), [dc], bpm, (j * run_bits, 0, 0))
            assert st is INVALID or st[0] % 2 == 1
        got, passes = parallel(intervals, [dc], bpm, run_bits)
        assert got == want and passes >= 2


def test_sync_model_invalid_codes_after_a_wrong_start():
    """An incomplete code (no codeword starts with 111) that the true path never meets: runs started at wrong
    boundaries run into it, end invalid, and the fix-up passes still recover the exact decode."""
    dc = {0: 2, 1: 2, 2: 3}                                   # 00, 01, 100   (101, 11x unused)
    ac = {0x00: 2, 0x01: 2, 0x11: 3, 0xF0: 4}                 # 00, 01, 100, 1010 (1011, 11xx unused)
    t = Tables(dc, ac)
    rng = random.Random(9)
    blocks = []
    for k in range(60):
        coefs = {0: rng.choice([0, 1, -1, 2, -3])}
        zz = 1
        while zz < 60 and rng.random() < 0.8:
            if rng.random() < 0.3:
                zz += 1
                if zz >= 64:
                    break
            coefs[zz] = rng.choice([1, -1])
            zz += 1
        blocks.append((0, coefs))
    # the value bits of size-1 coefficients can line up as 111 from a wrong start
    bits = encode(blocks, [t], rng)
    intervals = [(bits, 60)]
    want = sequential(intervals, [t], 1)
    saw_invalid = False
    for run_bits in (32, 41, 77, 128):
        n = -(-len(bits) // run_bits)
        for j in range(1, n):
            st, _ = decode_run(bits, min((j + 1) * run_bits, len(bits)), [t], 1, (j * run_bits, 0, 0))
            saw_invalid |= st is INVALID
        got, _ = parallel(intervals, [t], 1, run_bits)
        assert got == want
    assert saw_invalid

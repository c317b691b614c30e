"""Host side of the progressive JPEG decoder (csrc/jpeg.cu), no GPU: the parser's scan scripts and rejections, and a
Python model of the device's per-scan decode (the four scan kinds, EOB runs, restart intervals, the frame-MCU block
layout) that reproduces the quantised coefficients of each file's baseline-encoded twin.

Pillow only writes libjpeg's simple progression, so `custom_script_files` builds progressive files with a small
entropy encoder from the twin's coefficients: spectral selection only, non-interleaved DC, no DC successive
approximation, long EOB runs, Huffman tables redefined before every scan and a restart interval set between scans."""
import io
import random

import numpy as np
import pytest
from PIL import Image

from openibl_b200 import _cabi
from test_host_jpeg import canonical, extend, huff, take

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


# ---- a small marker reader -----------------------------------------------------------------------------------------

def _segments(data):
    """[(marker, payload)] up to and including each SOS; the entropy data follows as (None, destuffed intervals)."""
    out, i = [], 2
    while i < len(data):
        while data[i] == 0xFF and data[i + 1] == 0xFF:
            i += 1
        m = data[i + 1]
        if m == 0xD9:
            break
        ln = int.from_bytes(data[i + 2: i + 4], "big")
        out.append((m, data[i + 4: i + 2 + ln]))
        i += 2 + ln
        if m == 0xDA:
            ivs, cur = [], bytearray()
            while True:
                c = data[i]
                if c != 0xFF:
                    cur.append(c)
                    i += 1
                elif data[i + 1] == 0x00:
                    cur.append(0xFF)
                    i += 2
                elif data[i + 1] == 0xFF:
                    i += 1
                elif 0xD0 <= data[i + 1] <= 0xD7:
                    ivs.append(bytes(cur))
                    cur = bytearray()
                    i += 2
                else:
                    ivs.append(bytes(cur))
                    break
            out.append((None, ivs))
    return out


def _bits(b):
    return [(x >> (7 - k)) & 1 for x in b for k in range(8)]


def _table(counts, vals):
    code, out, p = 0, {}, 0
    for ln in range(1, 17):
        for _ in range(counts[ln - 1]):
            out[(ln, code)] = vals[p]
            p, code = p + 1, code + 1
        code <<= 1
    return out


def read_jpeg(data):
    """Frame and scans: {'w', 'h', 'comps': [(id, hs, vs)], 'scans': [{'comps', 'ss', 'se', 'ah', 'al', 'restart',
    'dc': {slot: table}, 'ac': {slot: table}, 'intervals': [bit lists]}]}."""
    f = {"scans": []}
    dc, ac, restart = {}, {}, 0
    segs = _segments(data)
    for k, (m, pl) in enumerate(segs):
        if m in (0xC0, 0xC1, 0xC2):
            f["h"], f["w"] = int.from_bytes(pl[1:3], "big"), int.from_bytes(pl[3:5], "big")
            f["comps"] = [(pl[6 + 3 * c], pl[7 + 3 * c] >> 4, pl[7 + 3 * c] & 15) for c in range(pl[5])]
            f["progressive"] = m == 0xC2
        elif m == 0xC4:
            i = 0
            while i < len(pl):
                tc, th = pl[i] >> 4, pl[i] & 15
                counts = list(pl[i + 1: i + 17])
                t = _table(counts, list(pl[i + 17: i + 17 + sum(counts)]))
                (dc if tc == 0 else ac)[th] = t
                i += 17 + sum(counts)
        elif m == 0xDD:
            restart = int.from_bytes(pl[:2], "big")
        elif m == 0xDA:
            ns = pl[0]
            ids = [c[0] for c in f["comps"]]
            comps = [ids.index(pl[1 + 2 * s]) for s in range(ns)]
            ss, se, a = pl[1 + 2 * ns], pl[2 + 2 * ns], pl[3 + 2 * ns]
            f["scans"].append({"comps": comps, "ss": ss, "se": se, "ah": a >> 4, "al": a & 15, "restart": restart,
                               "dc": {s: dc.get(pl[2 + 2 * s] >> 4) for s in range(ns)},
                               "ac": {s: ac.get(pl[2 + 2 * s] & 15) for s in range(ns)},
                               "intervals": [_bits(b) for b in segs[k + 1][1]]})
    return f


# ---- frame geometry and the block order of a scan --------------------------------------------------------------------

def geometry(f):
    comps = f["comps"] if len(f["comps"]) == 3 else [(f["comps"][0][0], 1, 1)]
    hmax, vmax = max(c[1] for c in comps), max(c[2] for c in comps)
    mx, my = -(-f["w"] // (8 * hmax)), -(-f["h"] // (8 * vmax))
    wb = [-(-f["w"] * c[1] // (8 * hmax)) for c in comps]
    hb = [-(-f["h"] * c[2] // (8 * vmax)) for c in comps]
    return comps, mx, my, wb, hb


def scan_blocks(f, sc):
    """[(scan component slot, component, block row, block column)] in the scan's order (jdinput.c per_scan_setup):
    MCU order with padding blocks when interleaved, the component's own raster otherwise."""
    comps, mx, my, wb, hb = geometry(f)
    if len(sc["comps"]) == 1:
        c = sc["comps"][0]
        return [(0, c, by, bx) for by in range(hb[c]) for bx in range(wb[c])]
    out = []
    for y in range(my):
        for x in range(mx):
            for slot, c in enumerate(sc["comps"]):
                _, hs, vs = comps[c]
                out += [(slot, c, y * vs + v, x * hs + h) for v in range(vs) for h in range(hs)]
    return out


def _intervals(f, sc):
    """The scan's blocks split into restart intervals of `restart` MCUs each."""
    blocks = scan_blocks(f, sc)
    comps = geometry(f)[0]
    bpm = 1 if len(sc["comps"]) == 1 else sum(comps[c][1] * comps[c][2] for c in sc["comps"])
    step = sc["restart"] * bpm if sc["restart"] else len(blocks)
    return [blocks[i: i + step] for i in range(0, len(blocks), step)]


def blank(f):
    comps, mx, my, wb, hb = geometry(f)
    return [np.zeros((my * vs, mx * hs, 64), np.int64) for _, hs, vs in comps]


# ---- sequential models of the decoders ------------------------------------------------------------------------------

def decode_baseline(f):
    """The twin's quantised coefficients, zig-zag order, per component on its MCU-padded block grid."""
    coef = blank(f)
    sc = f["scans"][0]
    for bits, blocks in zip(sc["intervals"], _intervals(f, sc)):
        pos, last = 0, [0, 0, 0]
        for slot, c, by, bx in blocks:
            s, ln = huff(sc["dc"][slot], bits, pos)
            last[slot] += extend(take(bits, pos + ln, s), s) if s else 0
            pos += ln + s
            coef[c][by, bx, 0] = last[slot]
            k = 1
            while k < 64:
                rs, ln = huff(sc["ac"][slot], bits, pos)
                r, s = rs >> 4, rs & 15
                pos += ln
                if s:
                    k += r
                    coef[c][by, bx, min(k, 63)] = extend(take(bits, pos, s), s)
                    pos += s
                    k += 1
                elif r == 15:
                    k += 16
                else:
                    break
    return coef


def _int16(v):
    return (v + 32768) % 65536 - 32768


def decode_progressive(f):
    """Model of the device's progressive path (csrc/jpeg.cu dc_first / jpeg_prog_dc_refine_kernel / ac_first /
    ac_refine): every scan in file order, every restart interval from its own start, EOB runs reset at each interval;
    raises on an invalid code, an interval that ends early or an EOB run past the interval's end."""
    coef = blank(f)
    for sc in f["scans"]:
        for bits, blocks in zip(sc["intervals"], _intervals(f, sc)):
            nbits, pos, eobrun, last = len(bits), 0, 0, [0, 0, 0]
            p1, m1 = 1 << sc["al"], -(1 << sc["al"])

            def need():
                if pos >= nbits:
                    raise ValueError("interval ends early")
            if sc["ss"] == 0 and sc["ah"] == 0:
                for slot, c, by, bx in blocks:
                    need()
                    s, ln = huff(sc["dc"][slot], bits, pos)
                    if s is None:
                        raise ValueError("invalid code")
                    last[slot] += extend(take(bits, pos + ln, s), s) if s else 0
                    pos += ln + s
                    coef[c][by, bx, 0] = _int16(last[slot] << sc["al"])
            elif sc["ss"] == 0:
                if len(blocks) > nbits:
                    raise ValueError("interval ends early")
                for t, (slot, c, by, bx) in enumerate(blocks):
                    if bits[t]:
                        coef[c][by, bx, 0] = _int16(coef[c][by, bx, 0] | p1)
            elif sc["ah"] == 0:
                for _, c, by, bx in blocks:
                    if eobrun:
                        eobrun -= 1
                        continue
                    k = sc["ss"]
                    while k <= sc["se"]:
                        need()
                        rs, ln = huff(sc["ac"][0], bits, pos)
                        if rs is None:
                            raise ValueError("invalid code")
                        r, s = rs >> 4, rs & 15
                        if s:
                            k += r
                            coef[c][by, bx, min(k, 63)] = _int16(extend(take(bits, pos + ln, s), s) << sc["al"])
                            pos += ln + s
                        elif r == 15:
                            k += 15
                            pos += ln
                        else:
                            eobrun = (1 << r) + take(bits, pos + ln, r) - 1
                            pos += ln + r
                            break
                        k += 1
            else:
                for _, c, by, bx in blocks:
                    blk = coef[c][by, bx]

                    def refine(z):
                        nonlocal pos
                        need()
                        if bits[pos] and (blk[z] & p1) == 0:
                            blk[z] = _int16(blk[z] + (p1 if blk[z] >= 0 else m1))
                        pos += 1
                    k = sc["ss"]
                    if eobrun == 0:
                        while k <= sc["se"]:
                            need()
                            rs, ln = huff(sc["ac"][0], bits, pos)
                            if rs is None or (rs & 15) > 1:
                                raise ValueError("invalid code")
                            r, s = rs >> 4, 0
                            pos += ln
                            if rs & 15:
                                need()
                                s = p1 if bits[pos] else m1
                                pos += 1
                            elif r != 15:
                                eobrun = (1 << r) + take(bits, pos, r)
                                pos += r
                                break
                            while k <= sc["se"]:
                                if blk[k] != 0:
                                    refine(k)
                                else:
                                    r -= 1
                                    if r < 0:
                                        break
                                k += 1
                            if s:
                                blk[min(k, 63)] = s
                            k += 1
                    if eobrun > 0:
                        while k <= sc["se"]:
                            if blk[k] != 0:
                                refine(k)
                            k += 1
                        eobrun -= 1
            if eobrun > 0:
                raise ValueError("EOB run past the end of the interval")
    return coef


def assert_same_coefficients(f, got, want):
    comps, mx, my, wb, hb = geometry(f)
    for c in range(len(comps)):
        np.testing.assert_array_equal(got[c][:hb[c], :wb[c]], want[c][:hb[c], :wb[c]], err_msg=f"component {c}")


# ---- a test-only progressive entropy encoder -----------------------------------------------------------------------

def _tables(seed, ac):
    """A full Huffman table with skewed lengths: every DC size, or every AC run/size, ZRL and EOBn symbol."""
    rng = random.Random(seed)
    if not ac:
        syms, lens = list(range(12)), [2, 3, 3, 3, 3, 3, 4, 5, 6, 7, 8, 9]
        rng.shuffle(syms)
    else:
        syms = [0xF0] + [r << 4 for r in range(15)] + [(r << 4) | s for r in range(16) for s in range(1, 11)]
        rng.shuffle(syms)
        lens = [3] * 4 + [5] * 6 + [7] * 10 + [10] * 10 + [16] * (len(syms) - 30)
    t = canonical(dict(zip(syms, lens)))
    return t, {s: lc for lc, s in t.items()}


def _dht(tc, th, t):
    items = sorted(t.items())                                  # by (length, code): canonical symbol order
    counts = [sum(1 for (ln, _c) in t if ln == L) for L in range(1, 17)]
    pl = bytes([(tc << 4) | th]) + bytes(counts) + bytes(s for _, s in items)
    return b"\xff\xc4" + (len(pl) + 2).to_bytes(2, "big") + pl


def _pack(bits):
    bits = bits + [1] * (-len(bits) % 8)
    out = bytearray()
    for i in range(0, len(bits), 8):
        v = int("".join(map(str, bits[i: i + 8])), 2)
        out.append(v)
        if v == 0xFF:
            out.append(0)
    return bytes(out)


def _value(v):
    s = int(abs(v)).bit_length()
    return s, (v if v > 0 else v + (1 << s) - 1)


def encode_scan(f, coef, comps, ss, se, ah, al, restart, seed):
    """DHT + DRI + SOS + entropy data of one scan (DC first / DC refinement / AC first, EOB runs up to 32767)."""
    sc = {"comps": comps, "restart": restart}
    dc, enc_dc = _tables(seed, False)
    ac, enc_ac = _tables(seed + 1, True)
    head = b""
    if ss == 0 and ah == 0:
        head += _dht(0, 0, dc)
    elif ss > 0:
        head += _dht(1, 0, ac)
    head += b"\xff\xdd\x00\x04" + restart.to_bytes(2, "big")
    ids = [c[0] for c in f["comps"]]
    pl = bytes([len(comps)]) + b"".join(bytes([ids[c], 0x00]) for c in comps) + bytes([ss, se, (ah << 4) | al])
    head += b"\xff\xda" + (len(pl) + 2).to_bytes(2, "big") + pl
    data = b""
    for n, blocks in enumerate(_intervals(f, sc)):
        bits, last, eobrun = [], [0, 0, 0], 0

        def put(lc, raw=None, s=0):
            ln, code = lc
            bits.extend((code >> (ln - 1 - i)) & 1 for i in range(ln))
            bits.extend((raw >> (s - 1 - i)) & 1 for i in range(s))

        def flush():
            nonlocal eobrun
            if eobrun:
                r = eobrun.bit_length() - 1
                put(enc_ac[r << 4], eobrun - (1 << r), r)
                eobrun = 0
        for slot, c, by, bx in blocks:
            z = coef[c][by, bx]
            if ss == 0 and ah == 0:
                v = int(z[0]) >> al
                s, raw = _value(v - last[slot])
                last[slot] = v
                put(enc_dc[s], raw, s)
            elif ss == 0:
                bits.append((int(z[0]) >> al) & 1)
            else:
                band = [int(z[k]) for k in range(ss, se + 1)]
                if not any(band):
                    eobrun += 1
                    if eobrun == 0x7FFF:
                        flush()
                    continue
                flush()
                r = 0
                for v in band:
                    if v == 0:
                        r += 1
                        continue
                    while r > 15:
                        put(enc_ac[0xF0])
                        r -= 16
                    s, raw = _value(v)
                    put(enc_ac[(r << 4) | s], raw, s)
                    r = 0
                if r:
                    eobrun += 1
                    if eobrun == 0x7FFF:
                        flush()
        flush()
        if n:
            data += bytes([0xFF, 0xD0 + (n - 1) % 8])
        data += _pack(bits)
    return head + data


# scripts as (components, Ss, Se, Ah, Al, restart interval)
SCRIPTS = {
    "spectral selection only": [((0, 1, 2), 0, 0, 0, 0, 0), ((0,), 1, 5, 0, 0, 0), ((1,), 1, 63, 0, 0, 0),
                                ((2,), 1, 63, 0, 0, 0), ((0,), 6, 20, 0, 0, 0), ((0,), 21, 63, 0, 0, 0)],
    "non-interleaved DC, DRI between scans": [((2,), 0, 0, 0, 1, 0), ((0,), 0, 0, 0, 1, 5), ((1,), 0, 0, 0, 1, 3),
                                              ((0, 1, 2), 0, 0, 1, 0, 2), ((0,), 1, 63, 0, 0, 7),
                                              ((1,), 1, 63, 0, 0, 0), ((2,), 1, 63, 0, 0, 1)],
    "one band per scan, long EOB runs": [((0, 1, 2), 0, 0, 0, 0, 0)] + [((c,), k, k, 0, 0, 0)
                                                                        for c in range(3) for k in range(1, 64)],
}


def progressive_file(twin, script, seed=0):
    """A progressive file with `script`, from the baseline twin's frame, quantisation tables and coefficients."""
    f = read_jpeg(twin)
    coef = decode_baseline(f)
    out = b"\xff\xd8"
    for m, pl in _segments(twin):
        if m in (0xDB,) or (m is not None and 0xE0 <= m <= 0xEF):
            out += bytes([0xFF, m]) + (len(pl) + 2).to_bytes(2, "big") + pl
        elif m == 0xC0:
            out += b"\xff\xc2" + (len(pl) + 2).to_bytes(2, "big") + pl
    ncomp = len(f["comps"])
    for i, (comps, ss, se, ah, al, restart) in enumerate(script):
        comps = tuple(c for c in comps if c < ncomp)
        if comps:
            out += encode_scan(f, coef, list(comps), ss, se, ah, al, restart, seed + 7 * i)
    return out + b"\xff\xd9"


def custom_script_files():
    """[(name, file)]: every custom script on colour (4:2:0, 4:4:4, 4:2:2) and grayscale images."""
    out = []
    for name, script in SCRIPTS.items():
        for j, (sub, mode) in enumerate([(2, "RGB"), (0, "RGB"), (1, "RGB"), (None, "L")]):
            kw = {} if sub is None else {"subsampling": sub}
            twin = _jpeg(_img(37 + 8 * j, 53 - 5 * j, 3 * j + len(name), mode), quality=75, **kw)
            out.append((f"{name} / {mode}{'' if sub is None else sub}", progressive_file(twin, script, seed=j)))
    return out


# ---- tests ----------------------------------------------------------------------------------------------------------

PILLOW_COLOUR = [((0, 1, 2), 0, 0, 0, 1), ((0,), 1, 5, 0, 2), ((2,), 1, 63, 0, 1), ((1,), 1, 63, 0, 1),
                 ((0,), 6, 63, 0, 2), ((0,), 1, 63, 2, 1), ((0, 1, 2), 0, 0, 1, 0), ((2,), 1, 63, 1, 0),
                 ((1,), 1, 63, 1, 0), ((0,), 1, 63, 1, 0)]
PILLOW_GRAY = [((0,), 0, 0, 0, 1), ((0,), 1, 5, 0, 2), ((0,), 6, 63, 0, 2), ((0,), 1, 63, 2, 1), ((0,), 0, 0, 1, 0),
               ((0,), 1, 63, 1, 0)]


@pytest.mark.parametrize("mode", ["RGB", "L"])
@pytest.mark.parametrize("extra", [{}, {"optimize": True}, {"restart_marker_blocks": 3}, {"restart_marker_rows": 1}])
def test_parser_accepts_pillow_progressive_files(mode, extra):
    data = _jpeg(_img(37, 53, 5, mode), quality=85, progressive=True, **extra)
    assert _cabi.jpeg_parse(data)["reason"] == "progressive"          # the baseline parser still refuses it
    info = _cabi.jpeg_parse_progressive(data)
    assert info["ok"], info["reason"]
    assert (info["width"], info["height"], info["components"]) == (53, 37, 3 if mode == "RGB" else 1)
    script = [(s["components"], s["ss"], s["se"], s["ah"], s["al"]) for s in info["scans"]]
    assert script == (PILLOW_COLOUR if mode == "RGB" else PILLOW_GRAY)
    assert info["intervals"] == sum(s["intervals"] for s in info["scans"])
    if extra.get("restart_marker_blocks") or extra.get("restart_marker_rows"):
        assert all(s["restart_interval"] > 0 for s in info["scans"]) and info["intervals"] > len(script)
    else:
        assert info["intervals"] == len(script)


def test_parser_rejects_sequential_files():
    info = _cabi.jpeg_parse_progressive(_jpeg(_img(16, 16, 1), quality=80))
    assert not info["ok"] and info["status"] == 6 and "not progressive" in info["reason"]


def _with_script(twin, script):
    return progressive_file(twin, [s + (0,) for s in script])


@pytest.mark.parametrize("script, reason", [
    ([((0, 1, 2), 0, 1, 0, 0)], "se != 0"),                                  # DC scan with Se > 0
    ([((0, 1, 2), 0, 0, 0, 0), ((0,), 5, 3, 0, 0)], "out of range"),         # Ss > Se
    ([((0, 1, 2), 0, 0, 0, 0), ((0, 1), 1, 63, 0, 0)], "more than one component"),
    ([((0, 1, 2), 0, 0, 0, 1), ((0, 1, 2), 0, 0, 2, 0)], "al != ah - 1"),
    ([((0, 1, 2), 0, 0, 0, 14)], "al > 13"),
    ([((0,), 1, 63, 0, 0)], "before the component's dc scan"),
    ([((0, 1, 2), 0, 0, 0, 2), ((0, 1, 2), 0, 0, 2, 1), ((0, 1, 2), 0, 0, 2, 1)], "previous al"),
])
def test_parser_rejects_bogus_scripts(script, reason):
    twin = _jpeg(_img(16, 24, 2), quality=80)
    # header only: the range checks run before any entropy data is read
    f = progressive_file(twin, [])[:-2]
    ids = [c[0] for c in read_jpeg(twin)["comps"]]
    for comps, ss, se, ah, al in script:
        pl = bytes([len(comps)]) + b"".join(bytes([ids[c], 0]) for c in comps) + bytes([ss, se, (ah << 4) | al])
        f += _dht(0, 0, _tables(0, False)[0]) + _dht(1, 0, _tables(1, True)[0])
        f += b"\xff\xda" + (len(pl) + 2).to_bytes(2, "big") + pl + b"\x00" * 4
    info = _cabi.jpeg_parse_progressive(f + b"\xff\xd9")
    assert not info["ok"] and info["status"] == 6, info
    assert reason in info["reason"].lower(), info["reason"]


@pytest.mark.parametrize("script", [
    [((0, 1, 2), 0, 0, 0, 0), ((0,), 1, 63, 0, 0), ((1,), 1, 63, 0, 0)],                 # Cr has no AC at all
    [((0, 1, 2), 0, 0, 0, 0), ((0,), 1, 5, 0, 1), ((1,), 1, 63, 0, 0), ((2,), 1, 63, 0, 0)],   # AC 1..5 not refined
    [((0, 1, 2), 0, 0, 0, 1), ((0,), 1, 63, 0, 0), ((1,), 1, 63, 0, 0), ((2,), 1, 63, 0, 0)],  # DC not refined
])
def test_parser_rejects_files_libjpeg_would_smooth(script):
    twin = _jpeg(_img(24, 32, 4), quality=80)
    info = _cabi.jpeg_parse_progressive(progressive_file(twin, [s + (0,) for s in script]))
    assert not info["ok"] and "smoothing" in info["reason"], info["reason"]
    # coefficients 10..63 may stay unrefined or uncoded: no smoothing, accepted
    ok = [((0, 1, 2), 0, 0, 0, 0)] + [((c,), 1, 9, 0, 0) for c in range(3)] + [((0,), 10, 63, 0, 1)]
    assert _cabi.jpeg_parse_progressive(progressive_file(twin, [s + (0,) for s in ok]))["ok"]


@pytest.mark.parametrize("sub", [0, 1, 2, "L"])
@pytest.mark.parametrize("extra", [{}, {"optimize": True}, {"restart_marker_blocks": 2}])
def test_model_reproduces_the_twins_coefficients_on_pillow_files(sub, extra):
    mode = "L" if sub == "L" else "RGB"
    kw = {} if sub == "L" else {"subsampling": sub}
    im = _img(29, 45, 11, mode)
    twin = read_jpeg(_jpeg(im, quality=90, **kw))
    prog = read_jpeg(_jpeg(im, quality=90, progressive=True, **kw, **extra))
    assert prog["progressive"] and not twin["progressive"]
    assert_same_coefficients(prog, decode_progressive(prog), decode_baseline(twin))


def test_model_reproduces_the_twins_coefficients_on_custom_scripts():
    files = custom_script_files()
    assert len(files) == 4 * len(SCRIPTS)
    for name, data in files:
        info = _cabi.jpeg_parse_progressive(data)
        assert info["ok"], (name, info["reason"])
        f = read_jpeg(data)
        got = decode_progressive(f)
        want = decode_baseline(read_jpeg(progressive_source(name)))
        assert_same_coefficients(f, got, want)


def progressive_source(name):
    """The baseline twin custom_script_files encoded `name` from."""
    script_name, kind = name.split(" / ")
    j = ["RGB2", "RGB0", "RGB1", "L"].index(kind)
    sub, mode = [(2, "RGB"), (0, "RGB"), (1, "RGB"), (None, "L")][j]
    kw = {} if sub is None else {"subsampling": sub}
    return _jpeg(_img(37 + 8 * j, 53 - 5 * j, 3 * j + len(script_name), mode), quality=75, **kw)


def test_custom_scripts_decode_like_their_twins_in_pillow():
    for name, data in custom_script_files():
        want = np.asarray(Image.open(io.BytesIO(progressive_source(name))).convert("RGB"))
        got = np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))
        assert np.array_equal(got, want), name


def test_model_reports_corrupt_streams():
    data = _jpeg(_img(29, 45, 12), quality=90, progressive=True)
    f = read_jpeg(data)
    sc = f["scans"][1]
    sc["intervals"][0] = sc["intervals"][0][: len(sc["intervals"][0]) // 3]
    with pytest.raises(ValueError, match="early"):
        decode_progressive(f)

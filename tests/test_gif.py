"""GIF decode (csrc/gif.cu): vips_gifload_buffer as nsgifload.c gives it, on the device and through its host twin.

The CPU half pins the host twin (the same per-code and per-pixel code the kernels run) to libnsgif itself: the oracle under
oracle/_ref restates nsgifload's header and generate over the reference's own gif.c and lzw.c.  Its inputs are the
reference test-suite's GIF fixtures (tests/golden/gif/) and a GIF writer of this file's own.  The GPU half pins the batch
decoder and the thumbnail entry points to the host twin and the oracle's thumbnail chain."""
import ctypes as C
import io
import os
import threading

import numpy as np
import pytest
from PIL import Image as PIL

import libvips_b200 as vb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "gif")
NSGIF = os.path.join(ROOT, "oracle", "_ref", "libnsgif_oracle.so")


# ---------------------------------------------------------------------------------------------------------- libnsgif

_nsgif = None


def nsgif():
    global _nsgif
    if _nsgif is None:
        if not os.path.exists(NSGIF):
            pytest.skip("oracle/_ref/libnsgif_oracle.so not built (needs the reference's libnsgif sources)")
        L = C.CDLL(NSGIF)
        L.nsgif_oracle_load.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_int), C.c_char_p, C.c_size_t]
        _nsgif = L
    return _nsgif


def oracle_load(s, page=0, n=1):
    """(pixels [h * pages, w, bands], None, scan result) or (None, message, scan result) as vips_gifload_buffer gives them"""
    L = nsgif()
    info = (C.c_int * 5)()
    msg = C.create_string_buffer(256)
    if L.nsgif_oracle_load(s, len(s), page, n, None, info, msg, 256):
        return None, msg.value.decode(), info[4]
    w, h, bands, fc, scan = info
    out = np.zeros((h * ((fc - page) if n == -1 else n), w, bands), np.uint8)
    if L.nsgif_oracle_load(s, len(s), page, n, out.ctypes.data, info, msg, 256):
        return None, msg.value.decode(), scan
    return out, None, scan


def twin(s, page=0, n=1):
    try:
        return vb.gif_decode_host_twin(s, page, n), None
    except vb.Error as e:
        return None, str(e)


def assert_pinned(s, page=0, n=1, declined=None):
    """the twin gives libnsgif's pixels; where nsgifload fails, or where its scan is not NSGIF_OK (declined), it refuses"""
    want, err, scan = oracle_load(s, page, n)
    got, gerr = twin(s, page, n)
    if want is None or scan != 0:
        assert got is None, (err, scan)
        if declined:
            assert declined in gerr, gerr
        return gerr
    assert got is not None, gerr
    assert got.shape == want.shape and np.array_equal(got, want)
    return got


# ---------------------------------------------------------------------------------------------------------- the writer

def pack_codes(codes, min_size):
    """LSB-first codes at the widths libnsgif reads them with (lzw.c:385-439: the width grows after the entry at the width's
    last code is added; a clear resets it; the first code after a clear adds nothing; the table stops at 4096)"""
    clear, eoi = 1 << min_size, (1 << min_size) + 1
    cs, ts, first = min_size + 1, eoi + 1, True
    acc = nbits = 0
    out = bytearray()
    for c in codes:
        acc |= c << nbits
        nbits += cs
        while nbits >= 8:
            out.append(acc & 255)
            acc >>= 8
            nbits -= 8
        if c == clear:
            cs, ts, first = min_size + 1, eoi + 1, True
        elif c == eoi:
            pass
        elif first:
            first = False
        elif ts < 4096:
            if ts == (1 << cs) - 1 and cs < 12:
                cs += 1
            ts += 1
    if nbits:
        out.append(acc & 255)
    return bytes(out)


def lzw_codes(indices, min_size, clear_at=None, eoi=True):
    """a plain LZW encoder: a clear when the table reaches clear_at (None: never, the table fills at 4096 and stays)"""
    clear = 1 << min_size
    codes = [clear]
    d, nxt = {}, clear + 2
    w = None
    for k in indices:
        k = int(k)
        if w is None:
            w = k
            continue
        if (w, k) in d:
            w = d[(w, k)]
            continue
        codes.append(w)
        if nxt < 4096:
            d[(w, k)] = nxt
            nxt += 1
        if clear_at and nxt >= clear_at:
            codes.append(clear)
            d, nxt = {}, clear + 2
        w = k
    if w is not None:
        codes.append(w)
    if eoi:
        codes.append(clear + 1)
    return codes


def interlace_order(h):
    return [y for start, step in ((0, 8), (4, 8), (2, 4), (1, 2)) for y in range(start, h, step)]


def sub_blocks(data, rng=None):
    out = bytearray()
    i = 0
    while i < len(data):
        n = 255 if rng is None else int(rng.integers(1, 256))
        out += bytes([len(data[i:i + n])]) + data[i:i + n]
        i += n
    return bytes(out) + b"\0"


def palette_bytes(pal):
    pal = np.asarray(pal, np.uint8).reshape(-1, 3)
    bits = max(1, int(np.ceil(np.log2(max(2, len(pal))))))
    full = np.zeros((1 << bits, 3), np.uint8)
    full[:len(pal)] = pal
    return bits - 1, full.tobytes()


def write_gif(W, H, frames, global_pal=None, bg=0, rng=None, trailer=True, head=b"GIF89a"):
    """frames: dicts with `img` (h x w indices, image rows), x, y, interlaced, local (palette), trans, disposal, min_size,
    clear_at, gce, and overrides: codes (raw code list), data (raw LZW bytes), tail (bytes after the codes)"""
    out = bytearray(head)
    flags = 0
    gt = b""
    if global_pal is not None:
        size, gt = palette_bytes(global_pal)
        flags = 0x80 | 0x70 | size
    out += bytes([W & 255, W >> 8, H & 255, H >> 8, flags, bg, 0]) + gt
    for f in frames:
        img = np.asarray(f["img"])
        h, w = img.shape
        trans, disposal = f.get("trans"), f.get("disposal", 0)
        if f.get("gce", True) and (trans is not None or disposal):
            out += bytes([0x21, 0xF9, 4, (disposal << 2) | (trans is not None), 10, 0, trans or 0, 0])
        fl = 0x40 if f.get("interlaced") else 0
        lt = b""
        if f.get("local") is not None:
            size, lt = palette_bytes(f["local"])
            fl |= 0x80 | size
        x, y = f.get("x", 0), f.get("y", 0)
        out += bytes([0x2C, x & 255, x >> 8, y & 255, y >> 8, w & 255, w >> 8, h & 255, h >> 8, fl]) + lt
        rows = img[interlace_order(h)] if f.get("interlaced") else img
        ms = f.get("min_size", 8)
        data = f.get("data")
        if data is None:
            codes = f.get("codes") or lzw_codes(rows.reshape(-1), ms, f.get("clear_at"))
            data = pack_codes(codes, ms)
        data += f.get("tail", b"")
        out += bytes([ms]) + sub_blocks(data, rng)
    if trailer:
        out += b"\x3B"
    return bytes(out)


def rand_pal(rng, n):
    return rng.integers(0, 256, (n, 3), dtype=np.uint8)


def noise(rng, h, w, colours):
    return rng.integers(0, colours, (h, w), dtype=np.int64)


def blocks(rng, h, w, colours, run=6):
    """photo-like enough: runs and repeats, so the table fills with long strings"""
    a = rng.integers(0, colours, (h // run + 1, w // run + 1)).repeat(run, 0).repeat(run, 1)[:h, :w]
    a[::5] = rng.integers(0, colours, (len(range(0, h, 5)), w))
    return a


# ---------------------------------------------------------------------------------------------------------- CPU: fixtures

FIXTURES = ["cogs", "cramps", "dispose-background", "dispose-previous", "invalid_multiframe", "trans-x", "truncated"]


def fixture(name):
    with open(os.path.join(GOLDEN, name + ".gif"), "rb") as f:
        return f.read()


@pytest.mark.parametrize("name", FIXTURES)
def test_fixtures_every_page(name):
    s = fixture(name)
    want, err, scan = oracle_load(s, 0, -1)
    if scan != 0:
        # nsgifload loads these only with a warning (truncated) or fails (invalid_multiframe): declined here
        with pytest.raises(vb.Error):
            vb.gif_decode_host_twin(s)
        return
    w, h, bands, frames = vb.gif_geometry(s)
    assert want.shape == (h * frames, w, bands)
    for page, n in [(0, 1), (0, -1), (frames // 2, 1), (frames // 2, -1), (frames - 1, 1)]:
        assert_pinned(s, page, n)
    for page in range(frames):
        assert np.array_equal(vb.gif_decode_host_twin(s, page, 1), want[page * h:(page + 1) * h])
    assert "bad page number" in twin(s, frames, 1)[1]
    assert "bad page number" in twin(s, 0, frames + 1)[1]
    assert "bad page number" in twin(s, -1, 1)[1]
    assert oracle_load(s, frames, 1)[1] == "bad page number"


def test_fixture_known_answers():
    """nsgifload's answers a reader can check by eye: trans-x has alpha, cramps has none"""
    assert vb.gif_geometry(fixture("trans-x"))[2] == 4
    assert vb.gif_geometry(fixture("cramps"))[:3] == (159, 203, 3)
    assert vb.gif_geometry(fixture("cogs"))[3] == 5


# ---------------------------------------------------------------------------------------------------------- CPU: the writer

def writer_cases():
    rng = np.random.default_rng(7)
    cases = {}
    for ms in range(2, 9):
        pal = rand_pal(rng, 1 << ms)
        cases["min%d_noise" % ms] = write_gif(23, 17, [dict(img=noise(rng, 17, 23, 1 << ms), min_size=ms)], pal, rng=rng)
        cases["min%d_blocks_clear" % ms] = write_gif(40, 31, [dict(img=blocks(rng, 31, 40, 1 << ms), min_size=ms, clear_at=200)], pal, rng=rng)
    pal = rand_pal(rng, 256)
    # no clears: the table fills at 4096 and stays
    cases["full_table"] = write_gif(200, 150, [dict(img=noise(rng, 150, 200, 37))], pal, rng=rng)
    cases["full_table_blocks"] = write_gif(211, 190, [dict(img=blocks(rng, 190, 211, 200, 3))], pal)
    cases["clear_4095"] = write_gif(120, 90, [dict(img=blocks(rng, 90, 120, 256, 2), clear_at=4095)], pal)
    # KwKwK: long runs of one value
    cases["kwkwk"] = write_gif(300, 7, [dict(img=np.full((7, 300), 3))], pal)
    cases["kwkwk_min2"] = write_gif(97, 41, [dict(img=np.where(np.arange(97 * 41).reshape(41, 97) % 211 < 200, 1, 2), min_size=2)], pal[:4])
    cases["interlaced"] = write_gif(31, 29, [dict(img=blocks(rng, 29, 31, 256), interlaced=True)], pal)
    for h in range(1, 10):
        cases["interlaced_h%d" % h] = write_gif(5, h, [dict(img=noise(rng, h, 5, 256), interlaced=True)], pal)
    cases["local_and_global"] = write_gif(30, 20, [dict(img=noise(rng, 20, 30, 256), local=rand_pal(rng, 256)),
                                                   dict(img=noise(rng, 10, 12, 4), x=3, y=4, local=rand_pal(rng, 4), min_size=2),
                                                   dict(img=noise(rng, 20, 30, 256))], pal)
    # indices past a small local table read what an earlier frame's larger local table left
    cases["stale_local"] = write_gif(16, 16, [dict(img=noise(rng, 16, 16, 256), local=rand_pal(rng, 256)),
                                              dict(img=noise(rng, 16, 16, 256), local=rand_pal(rng, 4))], pal)
    cases["no_global"] = write_gif(16, 9, [dict(img=noise(rng, 9, 16, 8), local=None, min_size=3)], None)
    cases["past_global"] = write_gif(16, 9, [dict(img=noise(rng, 9, 16, 16), min_size=4)], pal[:5])
    cases["transparency"] = write_gif(25, 20, [dict(img=noise(rng, 20, 25, 8), trans=3, min_size=3),
                                               dict(img=noise(rng, 8, 9, 8), x=2, y=5, trans=0, min_size=3)], pal[:8])
    for disp in (0, 1, 2, 3, 4, 5, 7):
        for t in (None, 1):
            fr = [dict(img=noise(rng, 20, 24, 8), min_size=3, disposal=disp if disp != 3 else 1),
                  dict(img=noise(rng, 7, 9, 8), x=5, y=6, trans=t, disposal=disp, min_size=3),
                  dict(img=noise(rng, 9, 6, 8), x=10, y=3, trans=2, disposal=disp, min_size=3),
                  dict(img=noise(rng, 4, 30, 8), x=0, y=15, disposal=2, min_size=3),
                  dict(img=noise(rng, 5, 5, 8), x=20, y=17, trans=4, min_size=3)]
            cases["disposal%d_t%s" % (disp, t)] = write_gif(24, 20, fr, pal[:8], bg=6, rng=rng)
    cases["bg_out_of_table"] = write_gif(12, 10, [dict(img=noise(rng, 10, 12, 4), min_size=2, disposal=2),
                                                  dict(img=noise(rng, 3, 3, 4), x=1, y=1, min_size=2)], pal[:4], bg=9)
    # offsets, clipping, a first frame that grows the screen, frames past the screen
    cases["offsets"] = write_gif(40, 30, [dict(img=noise(rng, 10, 10, 256), x=7, y=9),
                                          dict(img=noise(rng, 25, 30, 256), x=20, y=15),
                                          dict(img=noise(rng, 13, 17, 256), x=25, y=20, interlaced=True),
                                          dict(img=noise(rng, 5, 5, 256), x=41, y=2, disposal=2),
                                          dict(img=noise(rng, 5, 5, 256), x=2, y=31, disposal=2),
                                          dict(img=noise(rng, 30, 50, 256), x=0, y=0)], pal)
    cases["grows"] = write_gif(10, 10, [dict(img=noise(rng, 30, 20, 256), x=5, y=3), dict(img=noise(rng, 40, 40, 256), x=0, y=0)], pal)
    cases["broken_screen"] = write_gif(640, 480, [dict(img=noise(rng, 13, 11, 256), x=1, y=2)], pal)
    cases["big_screen"] = write_gif(3000, 20, [dict(img=noise(rng, 6, 7, 256))], pal)
    cases["full_width_offset_y"] = write_gif(20, 30, [dict(img=noise(rng, 12, 20, 256), y=25), dict(img=noise(rng, 12, 20, 256), y=4)], pal)
    # short data, early EOI, trailing data after EOI
    img = blocks(rng, 40, 50, 256)
    codes = lzw_codes(img.reshape(-1), 8)
    cases["short_data"] = write_gif(50, 40, [dict(img=img, data=pack_codes(codes[:len(codes) // 3], 8))], pal)
    cases["short_data_complex"] = write_gif(60, 40, [dict(img=img, x=3, data=pack_codes(codes[:len(codes) // 2], 8))], pal)
    cases["early_eoi"] = write_gif(50, 40, [dict(img=img, codes=codes[:len(codes) // 2] + [257] + codes[len(codes) // 2:])], pal)
    cases["early_eoi_interlaced"] = write_gif(50, 40, [dict(img=img, interlaced=True, codes=codes[:100] + [257])], pal)
    cases["trailing"] = write_gif(50, 40, [dict(img=img, tail=bytes(rng.integers(0, 256, 300, dtype=np.uint8)))], pal)
    cases["no_eoi"] = write_gif(50, 40, [dict(img=img, codes=codes[:-1])], pal)
    cases["only_clears"] = write_gif(5, 5, [dict(img=noise(rng, 5, 5, 4), codes=[4, 4, 4], min_size=2)], pal[:4])
    cases["empty_data"] = write_gif(5, 5, [dict(img=noise(rng, 5, 5, 4), data=b"", min_size=2)], pal[:4])
    cases["no_trailer"] = write_gif(9, 9, [dict(img=noise(rng, 9, 9, 256))], pal, trailer=False)
    cases["gif87a"] = write_gif(9, 9, [dict(img=noise(rng, 9, 9, 256))], pal, head=b"GIF87a")
    cases["one_by_one"] = write_gif(1, 1, [dict(img=np.array([[5]]))], pal)
    cases["one_by_one_min2"] = write_gif(1, 1, [dict(img=np.array([[1]]), min_size=2)], pal[:4])
    cases["min_code_9"] = write_gif(21, 13, [dict(img=noise(rng, 13, 21, 256), min_size=9)], pal)
    cases["min_code_11"] = write_gif(21, 13, [dict(img=noise(rng, 13, 21, 256), min_size=11)], pal)
    cases["tall_65535"] = write_gif(2, 65535, [dict(img=(np.arange(65535 * 2).reshape(65535, 2) // 7) % 256)], pal)
    cases["rows_65537"] = write_gif(1, 1, [dict(img=noise(rng, 65535, 1, 256), y=2)], pal)
    cases["animation"] = write_gif(33, 27, [dict(img=blocks(rng, 27, 33, 256), disposal=1)] +
                                   [dict(img=blocks(rng, 10 + k, 12, 256), x=k * 2, y=k, disposal=k % 4, trans=k * 3 if k % 2 else None)
                                    for k in range(7)], pal, bg=1, rng=rng)
    # extensions the walk skips
    plain = write_gif(9, 9, [dict(img=noise(rng, 9, 9, 256))], pal)
    ext = b"\x21\xFE\x05hello\x00" + b"\x21\xFF\x0BNETSCAPE2.0\x03\x01\x00\x00\x00" + b"\x21\x01\x0C" + bytes(12) + b"\x02ab\x00"
    cases["extensions"] = plain[:13 + 768] + ext + plain[13 + 768:]
    return cases


WRITER = writer_cases()


@pytest.mark.parametrize("name", sorted(WRITER))
def test_writer_pinned_to_libnsgif(name):
    s = WRITER[name]
    for page, n in [(0, 1), (0, -1)]:
        assert_pinned(s, page, n)
    frames = oracle_load(s, 0, 1)
    if frames[0] is not None:
        fc = vb.gif_geometry(s)[3]
        if fc > 2:
            assert_pinned(s, fc // 2, 2)


def test_writer_edge_geometry():
    g = vb.gif_geometry
    assert g(WRITER["grows"])[:2] == (25, 33)
    assert g(WRITER["broken_screen"])[:2] == (12, 15)
    assert g(WRITER["big_screen"])[:2] == (7, 6)
    assert g(WRITER["one_by_one"]) == (1, 1, 3, 1)
    assert g(WRITER["tall_65535"])[:2] == (2, 65535)
    with pytest.raises(vb.Error, match="bad image dimensions"):
        g(WRITER["rows_65537"])
    assert oracle_load(WRITER["rows_65537"])[0] is None


def test_pillow_agrees_on_static_frames():
    for name in ["min%d_noise" % ms for ms in range(2, 9)] + ["full_table", "full_table_blocks", "kwkwk", "interlaced", "clear_4095",
                                                               "min_code_9", "gif87a", "extensions"]:
        s = WRITER[name]
        got = vb.gif_decode_host_twin(s)
        assert got.shape[2] == 3
        im = PIL.open(io.BytesIO(s))
        assert np.array_equal(got, np.asarray(im.convert("RGB"))), name


# ---------------------------------------------------------------------------------------------------------- CPU: refusals

def bad_code_cases():
    rng = np.random.default_rng(3)
    pal = rand_pal(rng, 256)
    img = blocks(rng, 40, 50, 256)
    codes = lzw_codes(img.reshape(-1), 8)
    out = {}
    for at in (1, 2, 50, len(codes) // 2):
        past = 258 + (at - 1) + 1  # one past the table the decoder has when reading code `at`
        out["past_table_%d" % at] = write_gif(50, 40, [dict(img=img, codes=codes[:at] + [min(past, 511)] + codes[at:])], pal)
        out["past_table_%d_complex" % at] = write_gif(60, 40, [dict(img=img, x=2, codes=codes[:at] + [min(past, 511)] + codes[at:])], pal)
    out["first_code_eoi"] = write_gif(50, 40, [dict(img=img, codes=[256, 257])], pal)
    out["first_code_past_clear"] = write_gif(50, 40, [dict(img=img, codes=[256, 300])], pal)
    out["clear_then_eoi"] = write_gif(50, 40, [dict(img=img, codes=codes[:30] + [256, 257])], pal)
    out["clear_then_past"] = write_gif(50, 40, [dict(img=img, x=1, codes=codes[:30] + [256, 258])], pal)
    for ms in (0, 1, 12, 13, 59, 255):
        out["min_size_%d" % ms] = write_gif(8, 8, [dict(img=noise(rng, 8, 8, 2), data=bytes([0x55] * 40), min_size=ms)], pal)
    # the complex path: a bad code after exactly 4096 values is taken as the end of the frame, one value later it is not
    for extra in (0, 1, -1):
        n = 4096 + extra
        cs = [256]
        for v in range(n):  # a clear after every root code: one value per code
            cs += [v % 256, 256]
        for x in (0, 1):
            out["at_%d_x%d" % (n, x)] = write_gif(100 + x, 60, [dict(img=np.zeros((60, 100), np.int64), x=x, codes=cs[:-1] + [300])], pal)
    return out


BAD = bad_code_cases()


@pytest.mark.parametrize("name", sorted(BAD))
def test_refused_exactly_where_libnsgif_refuses(name):
    s = BAD[name]
    r = assert_pinned(s)
    want = oracle_load(s)
    if want[0] is None and want[2] == 0:
        # a frame libnsgif fails on, or (minimum code size 0x3B, the trailer byte) no frames at all
        assert want[1] in r or (want[1] == "Invalid frame data" and "bad LZW code" in r), (want[1], r)
    if name.startswith("at_4096_x1"):
        assert want[0] is not None  # the complex path's quiet end
    if name.startswith("at_4096_x0") or name.startswith("at_4097"):
        assert want[0] is None


def test_lzw_twin_alone():
    rng = np.random.default_rng(5)
    for ms in range(2, 9):
        idx = blocks(rng, 30, 41, 1 << ms).reshape(-1)
        for clear_at in (None, 300, 4095):
            data = pack_codes(lzw_codes(idx, ms, clear_at), ms)
            assert vb.lzw_host_twin(data, ms, idx.size) == bytes(idx.astype(np.uint8))
            assert vb.lzw_host_twin(data, ms, 100) == bytes(idx[:100].astype(np.uint8))
    # KwKwK from the first entry on
    data = pack_codes([4, 1, 6, 7, 5], 2)
    assert vb.lzw_host_twin(data, 2, 100) == bytes([1] * 6)
    with pytest.raises(vb.Error, match="bad LZW code"):
        vb.lzw_host_twin(pack_codes([4, 1, 7, 5], 2), 2, 100)
    with pytest.raises(vb.Error, match="minimum code size"):
        vb.lzw_host_twin(b"\0" * 4, 12, 10)
    # the last code needs a byte after it
    d = pack_codes([128, 65, 66], 7)
    assert len(d) == 3 and vb.lzw_host_twin(d, 7, 10) == b"A"
    assert vb.lzw_host_twin(d + b"\0", 7, 10) == b"AB"


def test_declines():
    rng = np.random.default_rng(9)
    pal = rand_pal(rng, 256)
    s = write_gif(20, 20, [dict(img=noise(rng, 20, 20, 256))] * 2, pal)
    cut = s[:len(s) - 40]
    assert oracle_load(cut)[0] is not None  # nsgifload promotes the cut frame and loads it
    with pytest.raises(vb.Error, match="truncated"):
        vb.gif_decode_host_twin(cut)
    with pytest.raises(vb.Error, match="not a GIF"):
        vb.gif_geometry(b"\x89PNG\r\n\x1a\n" + bytes(40))
    with pytest.raises(vb.Error, match="no frames"):
        vb.gif_geometry(s[:13 + 768] + b"\x3B")
    with pytest.raises(vb.Error, match="Invalid frame data"):
        vb.gif_geometry(s[:13 + 768] + b"\x99" + s[13 + 768:])


def test_abi_names():
    L = vb.lib()
    for name in ("vb200_gif_geometry", "vb200_gif_decode_batch", "vb200_gifload_buffer", "vb200_thumbnail_plan_run_gif",
                 "vb200_debug_gif_decode", "vb200_debug_lzw"):
        assert hasattr(L, name)


def test_batch_geometry_without_a_device():
    a, b = WRITER["transparency"], WRITER["animation"]
    w, h, bands = vb._gif_batch_geometry(vb.StreamBatch([a, a]), 0, -1)
    assert (w, h, bands) == (25, 40, 4)
    with pytest.raises(vb.Error, match="one geometry"):
        vb._gif_batch_geometry(vb.StreamBatch([a, b]), 0, 1)


# ---------------------------------------------------------------------------------------------------------- on the device

def animated(rng, W, H, nf, colours=256, trans=True, interlaced=False):
    pal = rand_pal(rng, 256)
    fr = [dict(img=blocks(rng, H, W, colours), disposal=1, local=rand_pal(rng, 256) if rng.integers(2) else None)]
    for k in range(1, nf):
        h, w = int(rng.integers(1, H + 1)), int(rng.integers(1, W + 1))
        fr.append(dict(img=blocks(rng, h, w, colours, 3), x=int(rng.integers(0, W - w + 1)), y=int(rng.integers(0, H - h + 1)),
                       disposal=int(rng.integers(0, 4)), trans=int(rng.integers(0, colours)) if trans and k == nf - 1 or rng.integers(3) == 0 else None,
                       interlaced=interlaced or bool(rng.integers(2)), local=rand_pal(rng, 256) if rng.integers(2) else None))
    fr[-1]["trans"] = fr[-1].get("trans") if not trans else 7
    return write_gif(W, H, fr, pal, bg=int(rng.integers(0, 256)), rng=rng)


def mixed(seed, n, W=37, H=29, nf=5):
    rng = np.random.default_rng(seed)
    return [animated(rng, W, H, nf) for _ in range(n)]


def _sentinel_decode(streams, shape, location, ptr, page=0, n=1):
    b = vb.StreamBatch(streams)
    _, h, w, bands = shape
    ww, hh, bb = C.c_int(), C.c_int(), C.c_int()
    return vb.lib().vb200_gif_decode_batch(b.ptrs, b.lens, b.n, page, n, C.c_void_p(ptr), location, w * bands, w * h * bands, C.byref(ww),
                                           C.byref(hh), C.byref(bb))


@pytest.mark.gpu
def test_gpu_mixed_batches(vb):
    import torch
    streams = mixed(1, 12)
    for page, n in [(0, 1), (0, -1), (2, 2), (4, 1)]:
        got = vb.gif_decode_batch(streams, page, n)
        for i, s in enumerate(streams):
            assert np.array_equal(got[i], vb.gif_decode_host_twin(s, page, n)), (page, n, i)
        w, h, bands = got.shape[2], got.shape[1], got.shape[3]
        bpl = w * bands + 3
        stride = bpl * h + 5
        dev = torch.full((stride * len(streams),), 77, dtype=torch.uint8, device="cuda")
        vb.gif_decode_batch(streams, page, n, out_ptr=dev.data_ptr(), out_bpl=bpl, out_frame_stride=stride)
        torch.cuda.synchronize()
        d = dev.cpu().numpy()
        for i in range(len(streams)):
            frame = d[i * stride:i * stride + bpl * h].reshape(h, bpl)
            assert np.array_equal(frame[:, :w * bands].reshape(h, w, bands), got[i]), (page, n, i)
            assert (frame[:, w * bands:] == 77).all()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(WRITER))
def test_gpu_writer_cases(vb, name):
    s = WRITER[name]
    try:
        want = vb.gif_decode_host_twin(s, 0, -1)
    except vb.Error:
        with pytest.raises(vb.Error):
            vb.gif_decode_batch([s], 0, -1)
        return
    assert np.array_equal(vb.gif_decode_batch([s, s], 0, -1)[1], want)


@pytest.mark.gpu
def test_gpu_fixtures_and_load_buffer(vb):
    for name in ("cogs", "cramps", "dispose-background", "dispose-previous", "trans-x"):
        s = fixture(name)
        want = vb.gif_decode_host_twin(s, 0, -1)
        assert np.array_equal(vb.gif_decode_batch([s, s], 0, -1)[1], want), name
        assert np.array_equal(vb.Image.gifload_buffer(s, 0, -1).numpy(), want), name
        assert np.array_equal(vb.Image.gifload_buffer(s).numpy(), vb.gif_decode_host_twin(s)), name


@pytest.mark.gpu
def test_gpu_70001_frames(vb):
    rng = np.random.default_rng(4)
    pal = rand_pal(rng, 256)
    ones = [write_gif(1, 1, [dict(img=np.array([[k]]), trans=5 if k % 2 else None)], pal) for k in range(4)]
    one = [ones[1], ones[3]]
    streams = [one[i % 2] for i in range(70001)]
    got = vb.gif_decode_batch(streams)
    for i in (0, 1, 65535, 65536, 70000):
        assert np.array_equal(got[i], vb.gif_decode_host_twin(streams[i])), i
    s = WRITER["tall_65535"]
    assert np.array_equal(vb.gif_decode_batch([s])[0], vb.gif_decode_host_twin(s))


@pytest.mark.gpu
@pytest.mark.parametrize("bad", ["code", "declined", "page"])
def test_gpu_batch_or_nothing(vb, bad):
    import torch
    streams = mixed(2, 9, nf=3)
    w, h, bands = vb._gif_batch_geometry(vb.StreamBatch(streams), 0, 1)
    want = vb.gif_decode_batch(streams)
    rng = np.random.default_rng(8)
    img = blocks(rng, h, w, 256)
    codes = lzw_codes(img.reshape(-1), 8)
    base = [dict(img=img, trans=3)]
    bad_stream = {
        "code": write_gif(w, h, [dict(img=img, trans=3, codes=codes[:40] + [511] + codes[40:])], rand_pal(rng, 256)),
        "declined": write_gif(w, h, base, rand_pal(rng, 256))[:-30],
        "page": write_gif(w, h, base[:1], rand_pal(rng, 256)),
    }[bad]
    k = 5
    batch = streams[:k] + [bad_stream] + streams[k:]
    L = vb.lib()
    pool = L.vb200_debug_dz_pool_used()
    shape = (len(batch), h, w, bands)
    out = np.full(shape, 0xA5, np.uint8)
    page = 1 if bad == "page" else 0
    rc = _sentinel_decode(batch, shape, vb.HOST, out.ctypes.data, page=page)
    msg = L.vb200_error_buffer().decode()
    L.vb200_error_clear()
    assert rc == -1 and "stream %d:" % k in msg, msg
    assert (out == 0xA5).all()
    dev = torch.full((int(np.prod(shape)),), 0xA5, dtype=torch.uint8, device="cuda")
    assert _sentinel_decode(batch, shape, vb.DEVICE, dev.data_ptr(), page=page) == -1
    L.vb200_error_clear()
    torch.cuda.synchronize()
    assert (dev.cpu().numpy() == 0xA5).all()
    assert L.vb200_debug_dz_pool_used() == pool
    assert np.array_equal(vb.gif_decode_batch(streams), want)
    assert L.vb200_debug_dz_pool_used() == pool


@pytest.mark.gpu
def test_gpu_chunks(vb):
    """batches split by the device-memory budget decode as one"""
    streams = mixed(3, 10, nf=4)
    want = vb.gif_decode_batch(streams, 0, -1)
    L = vb.lib()
    try:
        L.vb200_debug_png_set_budget(40000)
        assert np.array_equal(vb.gif_decode_batch(streams, 0, -1), want)
        L.vb200_debug_png_set_budget(100)
        with pytest.raises(vb.Error, match="more than the 100 allowed"):
            vb.gif_decode_batch(streams[:2])
    finally:
        L.vb200_debug_png_set_budget(0)


@pytest.mark.gpu
def test_gpu_two_threads(vb):
    import torch
    a, b = mixed(5, 16), mixed(6, 16)
    want = [vb.gif_decode_batch(a, 0, -1), vb.gif_decode_batch(b, 0, -1)]
    got = [None, None]

    def run(i, streams):
        torch.cuda.set_device(0)
        for _ in range(3):
            got[i] = vb.gif_decode_batch(streams, 0, -1)

    ts = [threading.Thread(target=run, args=(0, a)), threading.Thread(target=run, args=(1, b))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


def thumbnail_cases():
    rng = np.random.default_rng(12)
    pal = rand_pal(rng, 256)
    H, W = 300, 410
    rgb = write_gif(W, H, [dict(img=blocks(rng, H, W, 256, 10))], pal)
    rgba = write_gif(W, H, [dict(img=blocks(rng, H, W, 256, 10), trans=9), dict(img=blocks(rng, 50, 60, 256), x=9, y=9)], pal)
    return {"rgb": rgb, "rgba": rgba}


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["rgb", "rgba"])
def test_gpu_thumbnails(vb, oracle, case):
    s = thumbnail_cases()[case]
    dec = vb.gif_decode_host_twin(s)
    assert dec.shape[2] == (4 if case == "rgba" else 3)
    h, w, bands = dec.shape
    for target in (37, 128, 200):
        want = oracle.thumbnail_image(dec, target)
        assert np.array_equal(vb.thumbnail_buffer(s, target), want), (case, target)
        plan = vb.ThumbnailPlan(w, h, bands, target)
        got = plan.run_gif([s, s, s])
        plan.close()
        assert np.array_equal(got[2], want), (case, target)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["rgb", "rgba"])
def test_gpu_thumbnail_icc(vb, case):
    from icc_fixtures import rgb_profile
    s = thumbnail_cases()[case]
    out_prof = bytes(rgb_profile("srgb"))
    dec = vb.gif_decode_host_twin(s)
    want = vb.Image(dec).thumbnail_image(64, output_profile=out_prof).numpy()
    assert np.array_equal(vb.thumbnail_buffer(s, 64, output_profile=out_prof), want)
    want = vb.Image(dec).thumbnail_image_linear(64, output_profile=out_prof).numpy()
    assert np.array_equal(vb.thumbnail_buffer_linear(s, 64, output_profile=out_prof), want)
    want = vb.Image(dec).thumbnail_image_linear(64).numpy()
    assert np.array_equal(vb.thumbnail_buffer_linear(s, 64), want)
    plan = vb.ThumbnailPlan(dec.shape[1], dec.shape[0], dec.shape[2], 64)
    plan.set_icc(out_prof)
    got = plan.run_gif([s, s])
    plan.close()
    assert np.array_equal(got[1], vb.Image(dec).thumbnail_image(64, output_profile=out_prof).numpy())

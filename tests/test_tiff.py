"""TIFF load on the device (csrc/tiff.cu) against oracle/pytiff.py, and the oracle against Pillow's libtiff.

The streams come from a small TIFF 6.0 writer below (both byte orders, BigTIFF, strips and tiles with edge tiles and
short last strips, none / PackBits / LZW / deflate with and without predictor 2, pages, SubIFDs, ICCProfile), plus a few
that Pillow's libtiff writes.
"""
import io
import os
import struct
import zlib

import numpy as np
import pytest

import libvips_b200 as vb
from oracle import pyoracle, pytiff

PIL = pytest.importorskip("PIL.Image")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")

# ------------------------------------------------------------------ encoders (TIFF 6.0 sections 9, 13, 14; Adobe deflate)


def packbits_encode(b):
    out, i = bytearray(), 0
    while i < len(b):
        j = i
        while j + 1 < len(b) and b[j + 1] == b[i] and j - i < 127:
            j += 1
        if j > i:
            out += bytes([257 - (j - i + 1)]) + b[i:i + 1]
            i = j + 1
            continue
        j = i
        while j + 1 < len(b) and b[j + 1] != b[j] and j - i < 127:
            j += 1
        out += bytes([j - i]) + b[i:j + 1]
        i = j + 1
    return bytes(out)


def lzw_encode(b, clear_every=None):
    """libtiff's LZWEncode: MSB-first codes, a clear first, widening once the next free code passes 2^bits - 1, a clear when
    the table reaches 4094 (or every `clear_every` codes), the end code last"""
    out, acc, nacc = bytearray(), 0, 0
    nbits = 9

    def put(code):
        nonlocal acc, nacc
        acc = (acc << nbits) | code
        nacc += nbits
        while nacc >= 8:
            out.append((acc >> (nacc - 8)) & 255)
            nacc -= 8
        acc &= (1 << nacc) - 1

    put(256)
    table, free, emitted = {}, 258, 0
    w = None
    for c in b:
        if w is None:
            w = c
            continue
        key = (w, c)
        if key in table:
            w = table[key]
            continue
        put(w)
        emitted += 1
        table[key] = free
        free += 1
        w = c
        if free == 4094 or (clear_every and emitted % clear_every == 0):
            put(256)
            nbits, table, free = 9, {}, 258
        elif free > (1 << nbits) - 1:
            nbits += 1
    if w is not None:
        put(w)
        free += 1
        if free > (1 << nbits) - 1 and nbits < 12:
            nbits += 1
    put(257)
    if nacc:
        out.append((acc << (8 - nacc)) & 255)
    return bytes(out)


def difference(a):
    """predictor 2 over each row of a segment [rows, w, spp]"""
    d = a.astype(np.int16)
    d[:, 1:] -= a[:, :-1].astype(np.int16)
    return (d & 255).astype(np.uint8)


def encode(seg, comp, pred):
    if pred == 2 and comp in (5, 8, 32946):
        seg = difference(seg)
    raw = seg.tobytes()
    if comp == 1:
        return raw
    if comp == 32773:
        return packbits_encode(raw)
    if comp == 5:
        return lzw_encode(raw)
    return zlib.compress(raw, 6)


# ------------------------------------------------------------------ the writer


class Page:
    def __init__(self, img, photometric=None, comp=1, pred=1, tile=None, rps=None, extra=None, icc=None, orientation=None,
                 subifds=(), tags=None, segments=None):
        self.img = img if img.ndim == 3 else img[:, :, None]
        spp = self.img.shape[2]
        self.photometric = photometric if photometric is not None else (1 if spp < 3 else 2)
        self.comp, self.pred, self.tile, self.rps, self.icc = comp, pred, tile, rps, icc
        self.extra = extra if extra is not None else (2 if spp in (2, 4) else None)
        self.orientation, self.subifds, self.tags, self.segments = orientation, list(subifds), dict(tags or {}), segments


def _segments(p):
    a = p.img
    h, w, spp = a.shape
    if p.tile:
        tw, th = p.tile
        segs = []
        for y in range(0, h, th):
            for x in range(0, w, tw):
                t = np.zeros((th, tw, spp), np.uint8)
                part = a[y:y + th, x:x + tw]
                t[:part.shape[0], :part.shape[1]] = part
                segs.append(t)
        return segs
    rps = p.rps or h
    return [a[y:y + rps] for y in range(0, h, rps)]


def make_tiff(pages, order="<", big=False):
    buf = bytearray()
    cb, eb, inl = (8, 20, 8) if big else (2, 12, 4)
    off_type = 16 if big else 4

    def pack(fmt, *v):
        return struct.pack(order + fmt, *v)

    def align():
        if len(buf) & 1:
            buf.append(0)

    if big:
        buf += (b"II" if order == "<" else b"MM") + pack("HHHQ", 43, 8, 0, 0)
        first_at = 8
    else:
        buf += (b"II" if order == "<" else b"MM") + pack("HI", 42, 0)
        first_at = 4
    sizes = {3: ("H", 2), 4: ("I", 4), 16: ("Q", 8), 13: ("I", 4), 7: ("B", 1)}

    def write_ifd(p):
        data = p.segments if p.segments is not None else [encode(s, p.comp, p.pred) for s in _segments(p)]
        offs = []
        for d in data:
            align()
            offs.append(len(buf))
            buf.extend(d)
        subs = [write_ifd(s)[0] for s in p.subifds]
        h, w, spp = p.img.shape
        e = {256: (4, [w]), 257: (4, [h]), 258: (3, [8] * spp), 259: (3, [p.comp]), 262: (3, [p.photometric]), 277: (3, [spp]),
             284: (3, [1])}
        if p.pred != 1:
            e[317] = (3, [p.pred])
        if p.tile:
            e.update({322: (3, [p.tile[0]]), 323: (3, [p.tile[1]]), 324: (off_type, offs), 325: (off_type, [len(d) for d in data])})
        else:
            e.update({273: (off_type, offs), 278: (4, [p.rps or h]), 279: (off_type, [len(d) for d in data])})
        if p.extra is not None:
            e[338] = (3, [p.extra])
        if p.orientation is not None:
            e[274] = (3, [p.orientation])
        if p.icc is not None:
            e[34675] = (7, list(p.icc))
        if subs:
            e[330] = (off_type if big else 13, subs)
        e.update(p.tags)
        entries = []
        for tag in sorted(e):
            typ, vals = e[tag]
            f, sz = sizes[typ]
            payload = b"".join(pack(f, v) for v in vals)
            if len(payload) > inl:
                align()
                at = len(buf)
                buf.extend(payload)
                value = pack("Q" if big else "I", at)
            else:
                value = payload + b"\0" * (inl - len(payload))
            entries.append(pack("HH", tag, typ) + pack("Q" if big else "I", len(vals)) + value)
        align()
        at = len(buf)
        buf.extend(pack("Q" if big else "H", len(entries)))
        for x in entries:
            buf.extend(x)
        nxt = len(buf)
        buf.extend(b"\0" * (8 if big else 4))
        return at, nxt

    prev = first_at
    for p in pages:
        at, nxt = write_ifd(p)
        buf[prev:prev + (8 if big else 4)] = pack("Q" if big else "I", at)
        prev = nxt
    return bytes(buf)


def img(h, w, spp, seed=0, smooth=True):
    rng = np.random.default_rng(seed)
    if smooth:
        y, x = np.mgrid[0:h, 0:w]
        base = (x * 3 + y * 5)[:, :, None] + np.arange(spp) * 40
        return ((base + rng.integers(0, 6, (h, w, spp))) & 255).astype(np.uint8)
    return rng.integers(0, 256, (h, w, spp), dtype=np.uint8)


SOURCE = {}  # name -> the pixels the writer was given, as tiff2vips loads them


def _case(cases, name, pages, order="<", big=False):
    cases[name] = make_tiff(pages, order, big)
    a = pages[0].img.copy()
    if pages[0].photometric == 0:
        a[..., 0] = 255 - a[..., 0]
    SOURCE[name] = a


def stream_cases():
    """name -> stream, covering every layout and codec in scope"""
    cases = {}
    k = 0
    for comp in (1, 32773, 5, 8, 32946):
        for pred in ((1, 2) if comp in (5, 8, 32946) else (1,)):
            for spp, ph in ((1, 1), (1, 0), (2, 1), (3, 2), (4, 2)):
                for layout in ("strip", "tile"):
                    k += 1
                    a = img(37, 45, spp, k)
                    kw = dict(tile=(16, 16)) if layout == "tile" else dict(rps=7)
                    order = "<" if k % 2 else ">"
                    big = k % 3 == 0
                    name = "c%d-p%d-s%d-ph%d-%s-%s%s" % (comp, pred, spp, ph, layout, "le" if order == "<" else "be", "-big" if big else "")
                    _case(cases, name, [Page(a, ph, comp, pred, **kw)], order, big)
    _case(cases, "one-strip-lzw-noise", [Page(img(64, 48, 3, 99, smooth=False), comp=5)])
    _case(cases, "rps1-deflate", [Page(img(9, 30, 3, 5), comp=8, pred=2, rps=1)])
    _case(cases, "tile-larger-than-image", [Page(img(5, 7, 1, 6), comp=32773, tile=(16, 32))])
    _case(cases, "extra-unspecified", [Page(img(11, 13, 4, 7), comp=5, extra=0)])
    _case(cases, "icc", [Page(img(12, 12, 3, 8), comp=8, icc=bytes(range(256)) * 3)])
    return cases


def pillow_streams():
    out = {}
    a = img(33, 41, 3, 11)
    for comp in ("raw", "packbits", "tiff_lzw", "tiff_adobe_deflate"):
        b = io.BytesIO()
        PIL.fromarray(a).save(b, "TIFF", compression=comp)
        out["pillow-rgb-" + comp] = b.getvalue()
    for mode in ("L", "LA", "RGBA"):
        b = io.BytesIO()
        arr = img(21, 19, {"L": 1, "LA": 2, "RGBA": 4}[mode], 12)
        PIL.fromarray(arr[:, :, 0] if mode == "L" else arr, mode).save(b, "TIFF", compression="tiff_lzw")
        out["pillow-" + mode] = b.getvalue()
    return out


# ------------------------------------------------------------------ JPEG tiles (compression 7, TIFF Technical Note 2)

JPEG_TILES = {}  # name -> the tiles' pixels as Pillow's libjpeg-turbo decodes each complete JPEG before it is split


def _markers(j):
    """a JPEG stream's segments before SOS -> [(marker, bytes)], and the rest from SOS on"""
    out, p = [], 2
    while j[p + 1] != 0xDA:
        n = int.from_bytes(j[p + 2:p + 4], "big")
        out.append((j[p + 1], j[p:p + 2 + n]))
        p += 2 + n
    return out, j[p:]


def jpeg_tiles(a, tile, subsampling, tables, quality=85):
    """a [h, w, 1 or 3] cut into tiles, each a JPEG without JFIF (as libtiff writes them); with tables, every tile's DQT and
    DHT move to one JPEGTables stream (the first tile's: Pillow writes the same ones for every tile at one quality)
    -> (segments, JPEGTables or None, the pixels each complete tile decodes to, placed as the image)"""
    h, w, spp = a.shape
    tw, th = tile
    segs, table_bytes = [], None
    dec = np.zeros((-(-h // th) * th, -(-w // tw) * tw, spp), np.uint8)
    for y in range(0, h, th):
        for x in range(0, w, tw):
            t = np.zeros((th, tw, spp), np.uint8)
            part = a[y:y + th, x:x + tw]
            t[:part.shape[0], :part.shape[1]] = part
            b = io.BytesIO()
            im = PIL.fromarray(t[:, :, 0] if spp == 1 else t)
            im.save(b, "JPEG", quality=quality, **({} if spp == 1 else {"subsampling": subsampling}))
            full = b.getvalue()
            d = np.asarray(PIL.open(io.BytesIO(full)))
            dec[y:y + th, x:x + tw] = d if d.ndim == 3 else d[:, :, None]
            segments, rest = _markers(full)
            keep = [m for m in segments if m[0] != 0xE0]
            if tables:
                tab = b"".join(m[1] for m in keep if m[0] in (0xDB, 0xC4))
                table_bytes = table_bytes or b"\xff\xd8" + tab + b"\xff\xd9"
                keep = [m for m in keep if m[0] not in (0xDB, 0xC4)]
            segs.append(b"\xff\xd8" + b"".join(m[1] for m in keep) + rest)
    return segs, table_bytes, dec[:h, :w]


def jpeg_cases():
    cases = {}
    k = 0
    for spp, ph, sub in ((3, 6, 0), (3, 6, 1), (3, 6, 2), (1, 1, None), (1, 0, None)):
        for tables in (False, True):
            k += 1
            a = img(40, 50, spp, 60 + k)
            segs, tab, dec = jpeg_tiles(a, (16, 16), sub, tables)
            tags = {347: (7, list(tab))} if tables else {}
            name = "jpeg-s%d-ph%d-%s-%s" % (spp, ph, {0: "444", 1: "422", 2: "420", None: "grey"}[sub], "tables" if tables else "inline")
            cases[name] = make_tiff([Page(a, ph, comp=7, tile=(16, 16), segments=segs, tags=tags)], "<>"[k % 2], k % 3 == 0)
            if ph == 0:
                dec = dec.copy()
                dec[..., 0] = 255 - dec[..., 0]
            JPEG_TILES[name] = dec
    return cases


def padded_strip_case(cases):
    """deflate strips each holding RowsPerStrip rows, the last one padded past the image: libtiff reads what the image needs"""
    a = img(20, 13, 3, 71)
    pad = np.zeros((24, 13, 3), np.uint8)
    pad[:20] = a
    segs = [zlib.compress(pad[y:y + 8].tobytes()) for y in (0, 8, 16)]
    cases["deflate-padded-last-strip"] = make_tiff([Page(a, comp=8, rps=8, segments=segs)])
    SOURCE["deflate-padded-last-strip"] = a
    return cases


ALL = {**stream_cases(), **pillow_streams(), **jpeg_cases()}
padded_strip_case(ALL)


def pillow_load(s, page=0):
    im = PIL.open(io.BytesIO(s))
    im.seek(page)
    a = np.asarray(im)
    return a if a.ndim == 3 else a[:, :, None]


# ------------------------------------------------------------------ CPU


@pytest.mark.parametrize("name", sorted(ALL))
def test_oracle_matches_libtiff(name):
    """Pillow's libtiff where it opens the stream (it does not open big-endian tiled BigTIFF); the writer's own pixels too"""
    s = ALL[name]
    got = pytiff.load(s)
    if name in SOURCE:
        assert np.array_equal(got, SOURCE[name])
    if name in JPEG_TILES:
        # tiff2vips decodes JPEG tiles with its own libjpeg calls, not libtiff's JPEG codec: the evidence is that the spliced
        # tiles give what each complete JPEG gives
        assert np.array_equal(got, JPEG_TILES[name])
        return
    try:
        want = pillow_load(s)
    except PIL.UnidentifiedImageError:
        assert name.endswith("tile-be-big")
        return
    assert got.shape[:2] == want.shape[:2]
    b = min(got.shape[2], want.shape[2])
    assert np.array_equal(got[:, :, :b], want[:, :, :b])


@pytest.mark.parametrize("name", sorted(ALL))
def test_host_twin_matches_oracle(name):
    s = ALL[name]
    assert np.array_equal(vb.tiff_decode_host_twin(s), pytiff.load(s))


def test_geometry():
    s = make_tiff([Page(img(20, 30, 3, 1), comp=8, subifds=[Page(img(10, 15, 3, 2))]), Page(img(20, 30, 3, 3))], ">", True)
    assert vb.tiff_geometry(s) == (30, 20, 3, 2, 1)
    assert vb.tiff_geometry(s, 0, 0) == (15, 10, 3, 2, 1)
    assert vb.tiff_geometry(s, 1) == (30, 20, 3, 2, 0)


def test_pages_and_subifd_host_twin():
    p = [Page(img(16, 24, 1, i), comp=5, pred=2, tile=(16, 16), subifds=[Page(img(8, 12, 1, 10 + i), comp=32773)])
         for i in range(3)]
    s = make_tiff(p)
    for page, n, sub in ((0, 3, -1), (1, -1, -1), (2, 1, -1), (0, 2, 0), (1, 1, 0)):
        assert np.array_equal(vb.tiff_decode_host_twin(s, page, n, sub), pytiff.load(s, page, n, sub)), (page, n, sub)


def test_lzw_hook():
    rng = np.random.default_rng(5)
    for trial in range(60):
        n = int(rng.integers(1, 20000))
        kind = trial % 3
        if kind == 0:
            data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        elif kind == 1:
            data = rng.integers(0, 4, n, dtype=np.uint8).tobytes()
        else:
            data = bytes(rng.integers(0, 2, n, dtype=np.uint8) * 200)
        enc = lzw_encode(data, clear_every=int(rng.integers(50, 600)) if trial % 5 == 0 else None)
        assert pytiff.lzw_decode(enc, len(data)) == data
        assert vb.tiff_lzw_host_twin(enc, len(data)) == data
    # code-width boundaries: inputs whose tables end just around 511, 1023, 2047 and the 4094 clear
    for n in (250, 253, 254, 255, 256, 257, 508, 509, 510, 511, 512, 1020, 1021, 1022, 2044, 2045, 2046, 4091, 4093, 4094, 4095, 9000):
        data = bytes(range(256)) + bytes((i * 7 + i // 256) & 255 for i in range(n * 3))
        enc = lzw_encode(data)
        assert vb.tiff_lzw_host_twin(enc, len(data)) == pytiff.lzw_decode(enc, len(data)) == data
    # a clear right after a clear, then fewer bytes than asked for, then a first code that is not clear
    with pytest.raises(vb.Error, match="not enough data"):
        vb.tiff_lzw_host_twin(lzw_encode(b"abc"), 4)
    with pytest.raises(vb.Error, match="corrupt"):
        vb.tiff_lzw_host_twin(bytes([0x30, 0x80, 0x00]), 2)


def _pyramid_cases(rng, count):
    cases = []
    for i in range(count):
        w, h = int(rng.integers(8, 40000)), int(rng.integers(8, 40000))
        kind = i % 4
        n = int(rng.choice([0, 1, 2, 3, 5, 10, 27, 28, 29, 30]))
        jitter = lambda: int(rng.choice([0, 0, 1, -1, 5, -5, 6, -6]))
        if kind == 0:
            subs = [(w // (2 << k) + jitter(), h // (2 << k) + jitter()) for k in range(n)]
            pages = [(w, h)]
        elif kind == 1:
            subs = []
            pages = [(w // (1 << k) + (jitter() if k else 0), h // (1 << k) + (jitter() if k else 0)) for k in range(max(1, n))]
        elif kind == 2:
            subs = [(w // (2 << k), h // (2 << k)) for k in range(n)]
            pages = [(w // (1 << k), h // (1 << k)) for k in range(int(rng.integers(1, 6)))]
        else:
            subs = [(max(0, w // (2 << k) + jitter()), max(0, h // (2 << k) + jitter())) for k in range(n)]
            pages = [(w, h)] + [(int(rng.integers(1, 50)), int(rng.integers(1, 50))) for _ in range(int(rng.integers(0, 4)))]
        tw = int(rng.choice([1, 2, 64, 128, 256, 1000, 5000, 50000]))
        th = int(rng.choice([0, 1, 100, 256, 3000]))
        size = str(rng.choice(["both", "up", "down", "force"]))
        cases.append((w, h, pages, subs, tw, th, size))
    return cases


def test_pyramid_level_choice():
    rng = np.random.default_rng(2024)
    hits = set()
    for w, h, pages, subs, tw, th, size in _pyramid_cases(rng, 3000):
        got = vb.thumbnail_pyramid_level(w, h, pages, subs, tw, th or None, size)
        want = pytiff.pyramid_level(w, h, pages, subs, tw, th or None, size)
        assert got == want, (w, h, pages, subs, tw, th, size)
        hits.add((got[0] >= 0, got[1] > 0))
    assert hits == {(True, False), (False, True), (False, False)}
    # the edges: 5 px off is a level, 6 px is not; 2 px is a level, 1 px ends the search; 28 subifds / 29 pages at most
    assert vb.thumbnail_pyramid_level(1000, 1000, [(1000, 1000)], [(505, 500), (250, 245)], 100) == (1, 0)
    assert vb.thumbnail_pyramid_level(1000, 1000, [(1000, 1000)], [(506, 500), (250, 250)], 100) == (-1, 0)
    assert vb.thumbnail_pyramid_level(8, 8, [(8, 8)], [(4, 4), (2, 2)], 1) == (1, 0)
    assert vb.thumbnail_pyramid_level(4, 4, [(4, 4)], [(2, 2), (1, 1)], 1) == (-1, 0)
    big = 1 << 30
    subs = [(big // (2 << k), big // (2 << k)) for k in range(29)]
    assert vb.thumbnail_pyramid_level(big, big, [(big, big)], subs[:28], 1)[0] >= 0
    assert vb.thumbnail_pyramid_level(big, big, [(big, big)], subs, 1) == (-1, 0)
    pages = [(big >> k, big >> k) for k in range(30)]
    assert vb.thumbnail_pyramid_level(big, big, pages[:29], [], 1)[1] > 0
    assert vb.thumbnail_pyramid_level(big, big, pages, [], 1) == (-1, 0)


def pyramid_streams():
    base = img(256, 320, 3, 40)
    levels = [base[::1 << k, ::1 << k].copy() for k in range(4)]
    sub = make_tiff([Page(levels[0], comp=8, pred=2, tile=(64, 64), subifds=[Page(l, comp=5, tile=(32, 32)) for l in levels[1:]])])
    pages = make_tiff([Page(l, comp=8, tile=(32, 32)) for l in levels], ">")
    plain = make_tiff([Page(base, comp=5, rps=16)])
    return {"subifd": sub, "page": pages, "plain": plain}


@pytest.mark.parametrize("kind", ["subifd", "page", "plain"])
def test_tiff_level_hook(kind):
    s = pyramid_streams()[kind]
    w, h, pages, subs = pytiff.level_geometry(s)
    for tw in (10, 40, 70, 100, 159, 160, 161, 320, 500):
        assert vb.thumbnail_tiff_level(s, tw) == pytiff.pyramid_level(w, h, pages, subs, tw, None), tw


def declined_streams():
    a = img(8, 8, 1, 1)
    rgb = img(8, 8, 3, 1)
    return {
        "16-bit samples not supported": make_tiff([Page(a, tags={258: (3, [16])})]),
        "sample format 2 not supported": make_tiff([Page(a, tags={339: (3, [2])})]),
        "PlanarConfiguration 2": make_tiff([Page(rgb, tags={284: (3, [2])})]),
        "FillOrder 2 not supported": make_tiff([Page(a, tags={266: (3, [2])})]),
        "photometric 3 \\(palette\\)": make_tiff([Page(a, 3)]),
        "photometric 8 \\(CIELAB\\)": make_tiff([Page(rgb, 8)]),
        "photometric 5 \\(separated": make_tiff([Page(img(8, 8, 4, 1), 5, extra=None)]),
        "photometric 32844 \\(LogLuv\\)": make_tiff([Page(a, 32844)]),
        "YCbCr without JPEG": make_tiff([Page(rgb, 6)]),
        "JPEG-compressed strips not supported": make_tiff([Page(rgb, 6, comp=7, segments=[b"\xff\xd8\xff\xd9"])]),
        "RGB-photometric JPEG not supported": make_tiff([Page(rgb, 2, comp=7, tile=(16, 16), segments=[b"\xff\xd8\xff\xd9"])]),
        "tile 0: ": make_tiff([Page(rgb, 6, comp=7, tile=(16, 16), segments=[b"\xff\xd8\xff\xd9"])]),
        "JPEG tiles decode to 16 x 16 x 3, the IFD's tiles are 16 x 16 x 1": make_tiff([Page(
            a, 1, comp=7, tile=(16, 16), segments=jpeg_tiles(img(8, 8, 3, 1), (16, 16), 0, False)[0])]),
        "old-style JPEG": make_tiff([Page(rgb, comp=6, segments=[b"\xff\xd8\xff\xd9"])]),
        "associated alpha": make_tiff([Page(img(8, 8, 4, 1), extra=1)]),
        "compression 34712 not supported": make_tiff([Page(a, comp=34712, segments=[b"\0" * 64])]),
        "old-style LZW": make_tiff([Page(a, comp=5, segments=[b"\x00\x01\x02\x03"])]),
        "predictor 3 not supported": make_tiff([Page(a, comp=8, pred=3, segments=[zlib.compress(a.tobytes())])]),
        "lies outside the stream": make_tiff([Page(a, segments=[a.tobytes()], tags={273: (4, [1 << 20])})]),
        "pages cannot load as one strip": make_tiff([Page(a), Page(img(8, 9, 1, 2))]),
        "frames over 2\\^28 pixels": make_tiff([Page(a, segments=[a.tobytes()], tags={256: (4, [1 << 15]), 257: (4, [(1 << 13) + 1])})]),
        "greyscale with 3 samples": make_tiff([Page(rgb, 1)]),
        "not a TIFF stream": b"II\x2b\x00" + b"\0" * 20,
    }


@pytest.mark.parametrize("reason", list(declined_streams()))
def test_declined(reason):
    s = declined_streams()[reason]
    n = 2 if "one strip" in reason else 1
    with pytest.raises(vb.Error, match=reason):
        vb.tiff_decode_host_twin(s, 0, n)
    with pytest.raises(vb.Error, match=reason):  # the batch decoder's header pass, without a device
        vb._batch_geometry(vb.lib().vb200_tiff_decode_batch, [s], 0, n, -1)


def test_short_and_corrupt_segments():
    a = img(8, 8, 1, 3)
    short = {
        1: a.tobytes()[:60], 32773: packbits_encode(a.tobytes()[:60]), 5: lzw_encode(a.tobytes()[:60]),
        8: zlib.compress(a.tobytes()[:60]),
    }
    for comp, seg in short.items():
        s = make_tiff([Page(a, comp=comp, segments=[seg])])
        with pytest.raises(vb.Error):
            vb.tiff_decode_host_twin(s)
        with pytest.raises(ValueError):
            pytiff.load(s)
    # zlib checks the Adler-32 trailer when the last block ends with the rows full, and libtiff refuses a mismatch
    z = bytearray(zlib.compress(a.tobytes()))
    z[-1] ^= 1
    s = make_tiff([Page(a, comp=8, segments=[bytes(z)])])
    with pytest.raises(vb.Error, match="incorrect data check"):
        vb.tiff_decode_host_twin(s)
    with pytest.raises(zlib.error):
        pytiff.load(s)
    with pytest.raises(OSError, match="decoder error"):
        pillow_load(s)
    # without a trailer zlib waits for more input, and libtiff, its rows full, stops there
    s = make_tiff([Page(a, comp=8, segments=[zlib.compress(a.tobytes())[:-4]])])
    assert np.array_equal(vb.tiff_decode_host_twin(s), a) and np.array_equal(pytiff.load(s), a)
    assert np.array_equal(pillow_load(s), a)


def test_out_of_range_refused():
    """IFD offsets, entry counts, tag values and segments that point outside the stream are refused, never read"""
    s = make_tiff([Page(img(16, 16, 3, 4), comp=5, tile=(16, 16), subifds=[Page(img(8, 8, 3, 5))])])
    rng = np.random.default_rng(11)
    for i in range(400):
        b = bytearray(s)
        for _ in range(int(rng.integers(1, 4))):
            at = int(rng.integers(0, len(b)))
            b[at] = int(rng.integers(0, 256))
        if i % 4 == 0:
            b = b[:int(rng.integers(0, len(b)))]
        for fn in (lambda x: vb.tiff_decode_host_twin(x), lambda x: vb.tiff_geometry(x, 0, 0), lambda x: vb.tiff_icc_profile(x),
                   lambda x: vb.thumbnail_tiff_level(x, 4)):
            try:
                fn(bytes(b))
            except vb.Error:
                pass
    huge = bytearray(s)
    huge[4:8] = struct.pack("<I", 0xFFFFFFF0)
    with pytest.raises(vb.Error, match="outside the stream"):
        vb.tiff_geometry(bytes(huge))


def test_icc_and_orientation():
    prof = bytes(range(256)) * 5 + b"end"
    s = make_tiff([Page(img(6, 6, 3, 1), icc=prof, subifds=[Page(img(3, 3, 3, 2), icc=b"sub")])])
    assert vb.tiff_icc_profile(s) == prof == pytiff.icc_profile(s)
    assert vb.tiff_icc_profile(s, 0, 0) == b"sub"
    assert vb.tiff_icc_profile(make_tiff([Page(img(6, 6, 3, 1))])) is None


def test_pages_thumbnail_declines_tiff():
    s = make_tiff([Page(img(16, 16, 3, 1))])
    with pytest.raises(vb.Error, match="TIFF page strips"):
        vb.thumbnail_buffer(s, 8, return_page_height=True)


# ------------------------------------------------------------------ GPU


@pytest.mark.gpu
def test_decode_batch_every_stream():
    import torch
    for name, s in sorted(ALL.items()):
        want = pytiff.load(s)
        got = vb.tiff_decode_batch([s, s])
        assert np.array_equal(got[0], want) and np.array_equal(got[1], want), name
        h, w, b = want.shape
        bpl = w * b + 13
        stride = bpl * h + 29
        dev = torch.full((stride * 2,), 77, dtype=torch.uint8, device="cuda")
        vb.tiff_decode_batch([s, s], out_ptr=dev.data_ptr(), out_bpl=bpl, out_frame_stride=stride)
        torch.cuda.synchronize()
        host = dev.cpu().numpy()
        for f in range(2):
            fr = host[f * stride:f * stride + bpl * h].reshape(h, bpl)
            assert np.array_equal(fr[:, :w * b].reshape(h, w, b), want), name
            assert (fr[:, w * b:] == 77).all(), name
        assert (host[bpl * h:stride] == 77).all(), name


@pytest.mark.gpu
def test_mixed_batch_and_budget():
    a = img(40, 50, 3, 21)
    streams = [make_tiff([Page(a, comp=c, pred=p, **kw)], o, big)
               for c, p in ((1, 1), (32773, 1), (5, 2), (8, 1), (32946, 2), (5, 1))
               for kw in (dict(tile=(16, 16)), dict(rps=9))
               for o, big in (("<", False), (">", True))]
    for sub, tile in ((0, (16, 16)), (2, (16, 16)), (1, (32, 16))):  # JPEG tiles of two geometries: two JPEG batches per chunk
        segs, tab, _ = jpeg_tiles(a, tile, sub, True)
        streams.insert(3, make_tiff([Page(a, 6, comp=7, tile=tile, segments=segs, tags={347: (7, list(tab))})]))
    want = np.stack([pytiff.load(s) for s in streams])
    assert np.array_equal(want[0], a)
    assert np.array_equal(vb.tiff_decode_batch(streams), want)
    L = vb.lib()
    try:
        L.vb200_debug_png_set_budget(3 * 40 * 50 * 3)
        assert np.array_equal(vb.tiff_decode_batch(streams), want)
    finally:
        L.vb200_debug_png_set_budget(0)


@pytest.mark.gpu
def test_failing_stream_fails_batch():
    a = img(8, 8, 1, 3)
    good = make_tiff([Page(a, comp=5)])
    bad = make_tiff([Page(a, comp=5, segments=[lzw_encode(a.tobytes()[:50])])])
    with pytest.raises(vb.Error, match="frame 2: segment 0: not enough data"):
        vb.tiff_decode_batch([good, good, bad, good])
    corrupt = make_tiff([Page(a, comp=8, segments=[zlib.compress(a.tobytes())[:2] + b"\x07\x00" + b"\0" * 10])])
    with pytest.raises(vb.Error, match="frame 1: segment 0: corrupt"):
        vb.tiff_decode_batch([good, corrupt])
    z = bytearray(zlib.compress(a.tobytes()))
    z[-2] ^= 4
    with pytest.raises(vb.Error, match="frame 1: segment 0: incorrect data check"):
        vb.tiff_decode_batch([good, make_tiff([Page(a, comp=8, segments=[bytes(z)])])])
    rgb = img(16, 16, 3, 4)
    jgood = make_tiff([Page(rgb, 6, comp=7, tile=(16, 16), segments=jpeg_tiles(rgb, (16, 16), 2, False)[0])])
    seg = jpeg_tiles(rgb, (16, 16), 2, False)[0][0]
    jbad = make_tiff([Page(rgb, 6, comp=7, tile=(16, 16), segments=[seg[:len(seg) // 2]])])
    with pytest.raises(vb.Error, match="frame 1: tile 0: "):
        vb.tiff_decode_batch([jgood, jbad])


@pytest.mark.gpu
def test_pages_and_subifd():
    p = [Page(img(16, 24, 2, i), comp=8, pred=2, tile=(16, 16), subifds=[Page(img(8, 12, 2, 10 + i), comp=5, rps=3)]) for i in range(3)]
    s = make_tiff(p, ">", True)
    for page, n, sub in ((0, 3, -1), (1, -1, -1), (2, 1, -1), (0, 2, 0), (1, 1, 0)):
        want = pytiff.load(s, page, n, sub)
        assert np.array_equal(vb.tiff_decode_batch([s, s], page, n, sub)[1], want), (page, n, sub)
    im = vb.Image.tiffload_buffer(s, 0, 3)
    assert im.page_height == 16 and np.array_equal(im.numpy(), pytiff.load(s, 0, 3))


@pytest.mark.gpu
def test_tiffload_buffer():
    for prefix in ("c8-p2-s3-ph2-tile", "c5-p1-s1-ph0-strip", "pillow-RGBA"):
        name = next(k for k in sorted(ALL) if k.startswith(prefix))
        s = ALL[name]
        im = vb.Image.tiffload_buffer(s)
        assert np.array_equal(im.numpy(), pytiff.load(s)), name
        assert im.page_height is None


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["subifd", "page", "plain"])
def test_thumbnail_buffer_pyramids(kind):
    s = pyramid_streams()[kind]
    for tw in (40, 100, 159, 300):
        sub, page = vb.thumbnail_tiff_level(s, tw)
        level = pytiff.load(s, page, 1, sub)
        want = pyoracle.thumbnail_image(level, tw)
        assert np.array_equal(vb.thumbnail_buffer(s, tw), want), (kind, tw, sub, page)
    assert vb.thumbnail_tiff_level(s, 40) != (-1, 0) or kind == "plain"


@pytest.mark.gpu
def test_thumbnail_plan_run_tiff():
    a = img(64, 80, 4, 31)
    streams = [make_tiff([Page(a, comp=c, tile=(16, 16))]) for c in (5, 8, 32773)]
    plan = vb.ThumbnailPlan(80, 64, 4, 20)
    got = plan.run_tiff(streams)
    want = pyoracle.thumbnail_image(a, 20)
    for g in got:
        assert np.array_equal(g, want)


@pytest.mark.gpu
def test_thumbnail_embedded_profile_as_png():
    """an embedded ICCProfile drives colour management as PNG's iCCP does: the same pixels and profile give the same thumbnail"""
    prof = open(os.path.join(GOLDEN, "profiles", "p3.icm"), "rb").read()
    srgb = open(os.path.join(GOLDEN, "profiles", "sRGB.icm"), "rb").read()
    a = img(48, 64, 3, 33)
    t = make_tiff([Page(a, comp=8, icc=prof)])
    b = io.BytesIO()
    PIL.fromarray(a).save(b, "PNG", icc_profile=prof)
    want = vb.thumbnail_buffer(b.getvalue(), 20, output_profile=srgb)
    assert np.array_equal(vb.thumbnail_buffer(t, 20, output_profile=srgb), want)
    assert not np.array_equal(want, vb.thumbnail_buffer(make_tiff([Page(a, comp=8)]), 20, output_profile=srgb))
    with pytest.raises(vb.Error, match="Orientation 6"):
        vb.thumbnail_buffer(make_tiff([Page(a, orientation=6)]), 20)


@pytest.mark.gpu
def test_jpeg_tiled_thumbnail():
    a = img(96, 128, 3, 81)
    segs, tab, _ = jpeg_tiles(a, (32, 32), 2, True)
    s = make_tiff([Page(a, 6, comp=7, tile=(32, 32), segments=segs, tags={347: (7, list(tab))})])
    assert np.array_equal(vb.thumbnail_buffer(s, 40), pyoracle.thumbnail_image(pytiff.load(s), 40))


@pytest.mark.gpu
def test_plan_run_tiff_orientation_on_every_page():
    a = img(32, 32, 3, 91)
    s = make_tiff([Page(a, comp=8), Page(a, comp=8, orientation=6)])
    plan = vb.ThumbnailPlan(32, 32, 3, 8)
    assert np.array_equal(plan.run_tiff([s])[0], pyoracle.thumbnail_image(a, 8))
    with pytest.raises(vb.Error, match="Orientation 6"):  # page 1 of a two-page strip is not upright
        vb.ThumbnailPlan(32, 64, 3, 8, page_height=32).run_tiff([s], page=0, n=2)

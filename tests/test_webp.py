"""WebP load on the device (csrc/webp.cu): the host twin against the libwebp inside Pillow, then the device against the twin.

The streams come from Pillow's libwebp encoder (quality 0-100, method 0-6, photo-like, noise and flat content) and from a
seeded VP8 key-frame writer below, which reaches what Pillow's save options cannot: 2 / 4 / 8 token partitions, the simple
filter, every sharpness, levels 0 and 63, loop-filter deltas, segment maps with absolute and delta data, skip off,
probability updates, every 16x16, chroma and 4x4 mode (at frame edges too) and DCT_CAT6 coefficients.
"""
import ctypes as C
import glob
import io
import os
import struct
import threading

import numpy as np
import pytest

import libvips_b200 as vb

PIL = pytest.importorskip("PIL.Image")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "webp")


def pil_webp(a, **kw):
    b = io.BytesIO()
    PIL.fromarray(a).save(b, "WEBP", **kw)
    return b.getvalue()


def pillow(stream):
    return np.asarray(PIL.open(io.BytesIO(stream)).convert("RGB"))


def pillow_or_none(stream):
    try:
        im = PIL.open(io.BytesIO(stream))
        im.load()
        return np.asarray(im.convert("RGB"))
    except Exception:
        return None


def content(kind, h, w, seed):
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "flat":
        return np.broadcast_to(rng.integers(0, 256, 3, dtype=np.uint8), (h, w, 3)).copy()
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    a = np.stack([128 + 100 * np.sin(xx / 7 + yy / 13), 128 + 90 * np.cos(yy / 5 - xx / 17), (xx * 3 + yy * 2) % 256], -1)
    a += rng.normal(0, 6, a.shape)
    return np.clip(a, 0, 255).astype(np.uint8)


SIZES = [(1, 1), (15, 15), (16, 16), (17, 17), (31, 33), (33, 31), (16, 17), (7, 40), (120, 93), (211, 300)]


def pillow_streams():
    out = []
    for i, (h, w) in enumerate(SIZES):
        for j, kind in enumerate(("photo", "noise", "flat")):
            for q, m in ((0, 0), (15, 1), (30, 2), (75, 4), (60, 5), (95, 6), (100, 3)):
                if (i + j + q) % 2 and (h, w) not in ((1, 1), (17, 17)):
                    continue
                out.append(("%dx%d-%s-q%d-m%d" % (h, w, kind, q, m), pil_webp(content(kind, h, w, i * 7 + j), quality=q, method=m)))
    return out


PILLOW = pillow_streams()

# ------------------------------------------------------------------ a VP8 key-frame writer (RFC 6386)

T = vb.webp_tables() if os.path.exists(vb.library_path()) else None


def _tables():
    t = np.frombuffer(T, np.uint8)
    coeff0 = t[:1056].reshape(4, 8, 3, 11)
    upd = t[1056:2112].reshape(4, 8, 3, 11)
    bmodes = t[2112:3012].reshape(10, 10, 9)
    dc = t[3012:3140]
    ac = np.frombuffer(T[3140:3396], "<u2")
    zigzag = t[3396:3412]
    bands = t[3412:3429]
    return coeff0, upd, bmodes, dc, ac, zigzag, bands


CAT = [[173, 148, 140], [176, 155, 140, 135], [180, 157, 141, 134, 130], [254, 254, 243, 230, 196, 177, 153, 140, 133, 130, 129]]


class BoolEnc:
    """the boolean entropy encoder of RFC 6386 7.3"""

    def __init__(self):
        self.out, self.range, self.bottom, self.bit_count = bytearray(), 255, 0, 24

    def put(self, bit, prob):
        split = 1 + (((self.range - 1) * prob) >> 8)
        if bit:
            self.bottom += split
            self.range -= split
        else:
            self.range = split
        while self.range < 128:
            self.range <<= 1
            if self.bottom & (1 << 31):
                i = len(self.out) - 1
                while self.out[i] == 255:
                    self.out[i] = 0
                    i -= 1
                self.out[i] += 1
            self.bottom = (self.bottom << 1) & 0xFFFFFFFF
            self.bit_count -= 1
            if self.bit_count == 0:
                self.out.append(self.bottom >> 24)
                self.bottom &= 0xFFFFFF
                self.bit_count = 8

    def value(self, v, n):
        for k in range(n - 1, -1, -1):
            self.put((v >> k) & 1, 128)

    def signed(self, v, n):
        self.value(abs(v), n)
        self.put(v < 0, 128)

    def flag_signed(self, v, n):
        self.put(v != 0, 128)
        if v:
            self.signed(v, n)

    def finish(self):
        for _ in range(32):
            self.put(0, 128)
        return bytes(self.out)


DC_, TM_, VE_, HE_ = 0, 1, 2, 3
# sub-block mode -> its path through the tree: (bit, probability index)
BPATH = {0: [(0, 0)], 1: [(1, 0), (0, 1)], 2: [(1, 0), (1, 1), (0, 2)], 3: [(1, 0), (1, 1), (1, 2), (0, 3), (0, 4)],
         4: [(1, 0), (1, 1), (1, 2), (0, 3), (1, 4), (0, 5)], 5: [(1, 0), (1, 1), (1, 2), (0, 3), (1, 4), (1, 5)],
         6: [(1, 0), (1, 1), (1, 2), (1, 3), (0, 6)], 7: [(1, 0), (1, 1), (1, 2), (1, 3), (1, 6), (0, 7)],
         8: [(1, 0), (1, 1), (1, 2), (1, 3), (1, 6), (1, 7), (0, 8)], 9: [(1, 0), (1, 1), (1, 2), (1, 3), (1, 6), (1, 7), (1, 8)]}
YPATH = {DC_: [(0, 156), (0, 163)], VE_: [(0, 156), (1, 163)], HE_: [(1, 156), (0, 128)], TM_: [(1, 156), (1, 128)]}
UVPATH = {DC_: [(0, 142)], VE_: [(1, 142), (0, 114)], TM_: [(1, 142), (1, 114), (1, 183)], HE_: [(1, 142), (1, 114), (0, 183)]}


def put_level(e, p, v):
    """|v| >= 2 through the large-value tree; p: the band / context probabilities"""
    if v <= 4:
        e.put(0, p[3])
        e.put(v > 2, p[4])
        if v > 2:
            e.put(v - 3, p[5])
    elif v <= 10:
        e.put(1, p[3])
        e.put(0, p[6])
        e.put(v > 6, p[7])
        if v <= 6:
            e.put(v - 5, 159)
        else:
            e.put((v - 7) >> 1, 165)
            e.put((v - 7) & 1, 145)
    else:
        e.put(1, p[3])
        e.put(1, p[6])
        cat = 0 if v < 19 else 1 if v < 35 else 2 if v < 67 else 3
        e.put(cat >> 1, p[8])
        e.put(cat & 1, p[9 + (cat >> 1)])
        extra, nb = v - (3 + (8 << cat)), len(CAT[cat])
        for k, pr in enumerate(CAT[cat]):
            e.put((extra >> (nb - 1 - k)) & 1, pr)


def put_block(e, proba, bands, ctx, first, levels):
    """levels in zigzag order; returns whether the block has a coefficient at or past `first` (the neighbours' context)"""
    nzs = [k for k in range(first, 16) if levels[k]]
    last = nzs[-1] if nzs else -1
    n, p = first, proba[bands[first]][ctx]
    while n < 16:
        if n > last:
            e.put(0, p[0])
            return last >= first
        e.put(1, p[0])
        while levels[n] == 0:
            e.put(0, p[1])
            n += 1
            p = proba[bands[n]][0]
        e.put(1, p[1])
        v = abs(int(levels[n]))
        if v == 1:
            e.put(0, p[2])
            nctx = 1
        else:
            e.put(1, p[2])
            put_level(e, p, v)
            nctx = 2
        e.put(levels[n] < 0, 128)
        n += 1
        p = proba[bands[n]][nctx]
    return last >= first


def vp8_stream(seed, h=None, w=None, parts=None, simple=None, level=None, sharp=None, skip=None, segments=None, lf_delta=None,
               updates=None, cat6=False, mode=None):
    """one seeded key frame as a simple-format WebP stream; each unset option is drawn from the seed"""
    coeff0, upd, bmodes, dc, ac, zigzag, bands = _tables()
    r = np.random.default_rng(seed)
    pick = lambda v, f: f() if v is None else v  # noqa: E731
    h = pick(h, lambda: int(r.integers(1, 70)))
    w = pick(w, lambda: int(r.integers(1, 70)))
    parts = pick(parts, lambda: int(r.choice([1, 2, 4, 8])))
    simple = pick(simple, lambda: bool(r.integers(0, 2)))
    level = pick(level, lambda: int(r.choice([0, 1, 10, 20, 40, 63, int(r.integers(0, 64))])))
    sharp = pick(sharp, lambda: int(r.integers(0, 8)))
    skip = pick(skip, lambda: bool(r.integers(0, 2)))
    segments = pick(segments, lambda: int(r.integers(0, 3)))  # 0 none, 1 absolute, 2 delta
    lf_delta = pick(lf_delta, lambda: bool(r.integers(0, 2)))
    updates = pick(updates, lambda: bool(r.integers(0, 2)))
    mb_w, mb_h = (w + 15) // 16, (h + 15) // 16
    e = BoolEnc()
    e.put(0, 128)
    e.put(int(r.integers(0, 2)), 128)
    e.put(segments > 0, 128)
    seg_p = [255, 255, 255]
    base_q = int(r.integers(0, 40)) if not cat6 else 0
    seg_q = [0, 0, 0, 0]
    if segments:
        e.put(1, 128)  # update map
        e.put(1, 128)  # update data
        e.put(segments == 1, 128)
        seg_q = [int(r.integers(0, 30)) if segments == 1 else int(r.integers(-10, 20)) for _ in range(4)]
        for q in seg_q:
            e.flag_signed(q, 7)
        for _ in range(4):
            e.flag_signed(int(r.integers(-63, 64)) if r.integers(0, 2) else 0, 6)
        seg_p = [int(x) for x in r.integers(0, 256, 3)]
        for p in seg_p:
            e.put(1, 128)
            e.value(p, 8)
    e.put(simple, 128)
    e.value(level, 6)
    e.value(sharp, 3)
    e.put(lf_delta, 128)
    if lf_delta:
        e.put(1, 128)
        for _ in range(8):
            e.flag_signed(int(r.integers(-63, 64)) if r.integers(0, 2) else 0, 6)
    e.value({1: 0, 2: 1, 4: 2, 8: 3}[parts], 2)
    e.value(base_q, 7)
    for _ in range(5):
        e.flag_signed(int(r.integers(-15, 16)) if r.integers(0, 3) == 0 else 0, 4)
    e.put(0, 128)  # refresh entropy probs
    proba = coeff0.astype(np.int64).copy()
    for idx in np.ndindex(4, 8, 3, 11):
        if updates and r.integers(0, 12) == 0:
            e.put(1, int(upd[idx]))
            proba[idx] = int(r.integers(1, 256))
            e.value(int(proba[idx]), 8)
        else:
            e.put(0, int(upd[idx]))
    skip_p = int(r.integers(1, 255))
    e.put(skip, 128)
    if skip:
        e.value(skip_p, 8)
    # macroblocks
    toks = [BoolEnc() for _ in range(parts)]
    top_modes = np.zeros((mb_w, 4), int)
    top_nz, top_dc = np.zeros(mb_w, int), np.zeros(mb_w, int)
    for my in range(mb_h):
        left_modes = [0, 0, 0, 0]
        lnz, ldc = 0, 0
        te = toks[my % parts]
        for mx in range(mb_w):
            seg = int(r.integers(0, 4))
            if segments:
                e.put(seg >= 2, seg_p[0])
                e.put(seg & 1, seg_p[1 + (seg >> 1)])
            else:
                seg = 0
            sk = skip and r.integers(0, 4) == 0
            if skip:
                e.put(sk, skip_p)
            i4 = bool(r.integers(0, 2)) if mode is None else mode == "i4"
            e.put(not i4, 145)
            if not i4:
                ym = int(r.integers(0, 4))
                for b, p in YPATH[ym]:
                    e.put(b, p)
                top_modes[mx, :] = ym
                left_modes = [ym] * 4
            else:
                for y in range(4):
                    for x in range(4):
                        bm = int(r.integers(0, 10))
                        pr = bmodes[top_modes[mx, x], left_modes[y]]
                        for b, i in BPATH[bm]:
                            e.put(b, int(pr[i]))
                        top_modes[mx, x] = bm
                        left_modes[y] = bm
            for b, p in UVPATH[int(r.integers(0, 4))]:
                e.put(b, p)
            if sk:
                top_nz[mx] = lnz = 0
                if not i4:
                    top_dc[mx] = ldc = 0
                continue

            def levels(limit, density):
                lv = np.zeros(16, int)
                if r.integers(0, 3):
                    k = r.random(16) < density
                    lv[k] = r.integers(1, limit + 1, int(k.sum())) * np.where(r.random(int(k.sum())) < 0.5, -1, 1)
                return lv

            big = 500 if cat6 else 30
            if not i4:
                has = put_block(te, proba[1], bands, top_dc[mx] + ldc, 0, levels(big if cat6 else 12, 0.3))
                top_dc[mx] = ldc = int(has)
                first, pt = 1, proba[0]
            else:
                first, pt = 0, proba[3]
            tn, ln = top_nz[mx], lnz
            new_t, new_l = 0, 0
            tcol = [(tn >> x) & 1 for x in range(4)]
            for y in range(4):
                lbit = (ln >> y) & 1
                for x in range(4):
                    has = int(put_block(te, pt, bands, lbit + tcol[x], first, levels(big, 0.25)))
                    lbit = tcol[x] = has
                new_l |= lbit << y
            new_t = sum(tcol[x] << x for x in range(4))
            for ch in (0, 1):
                tcol = [(tn >> (4 + 2 * ch + x)) & 1 for x in range(2)]
                for y in range(2):
                    lbit = (ln >> (4 + 2 * ch + y)) & 1
                    for x in range(2):
                        has = int(put_block(te, proba[2], bands, lbit + tcol[x], 0, levels(big, 0.25)))
                        lbit = tcol[x] = has
                    new_l |= lbit << (4 + 2 * ch + y)
                new_t |= sum(tcol[x] << (4 + 2 * ch + x) for x in range(2))
            top_nz[mx], lnz = new_t, new_l
    p0 = e.finish()
    tp = [t.finish() for t in toks]
    sizes = b"".join(struct.pack("<I", len(t))[:3] for t in tp[:-1])
    tag = (0 | (0 << 1) | (1 << 4) | (len(p0) << 5))
    vp8 = struct.pack("<I", tag)[:3] + b"\x9d\x01\x2a" + struct.pack("<HH", w, h) + p0 + sizes + b"".join(tp)
    return riff([(b"VP8 ", vp8)])


def riff(chunks):
    body = b"WEBP"
    for tag, data in chunks:
        body += tag + struct.pack("<I", len(data)) + data + (b"\0" if len(data) & 1 else b"")
    return b"RIFF" + struct.pack("<I", len(body)) + body


def vp8_payload(stream):
    """the VP8 chunk of a simple-format stream"""
    assert stream[12:16] == b"VP8 "
    n = struct.unpack("<I", stream[16:20])[0]
    return stream[20:20 + n]


def writer_streams():
    out = []
    for parts in (1, 2, 4, 8):
        out.append(("parts%d" % parts, vp8_stream(100 + parts, h=70, w=40, parts=parts)))
    for sharp in range(8):
        for simple in (False, True):
            out.append(("sharp%d-simple%d" % (sharp, simple), vp8_stream(200 + sharp * 2 + simple, sharp=sharp, simple=simple, level=30)))
    for level in (0, 1, 63):
        out.append(("level%d" % level, vp8_stream(300 + level, level=level)))
    for segments in (0, 1, 2):
        for lf in (False, True):
            out.append(("seg%d-lf%d" % (segments, lf), vp8_stream(400 + segments * 2 + lf, segments=segments, lf_delta=lf)))
    out.append(("skip-off", vp8_stream(500, skip=False)))
    out.append(("skip-on", vp8_stream(501, skip=True)))
    out.append(("updates", vp8_stream(502, updates=True)))
    out.append(("i4-edges", vp8_stream(503, h=33, w=47, mode="i4")))
    out.append(("i16-edges", vp8_stream(504, h=17, w=1, mode="i16")))
    out.append(("cat6", vp8_stream(505, cat6=True, h=40, w=40)))
    for s in range(200):
        out.append(("random%d" % s, vp8_stream(1000 + s)))
    return out


WRITER = writer_streams() if T is not None else []

# ------------------------------------------------------------------ CPU: the host twin against libwebp


def test_tables_are_libwebps():
    """every constant table, as one array, appears verbatim in the libwebp shared object Pillow loads"""
    import PIL as P
    found = glob.glob(os.path.join(os.path.dirname(P.__file__), "..", "pillow.libs", "libwebp-*.so*"))
    if not found:
        pytest.skip("no bundled libwebp to search")
    so = open(found[0], "rb").read()
    sizes = [("coefficient defaults", 1056), ("coefficient updates", 1056), ("sub-block modes", 900), ("dc", 128), ("ac", 256),
             ("zigzag", 16), ("bands", 17)]
    at = 0
    for name, n in sizes:
        assert so.find(T[at:at + n]) >= 0, name
        at += n


@pytest.mark.parametrize("name,stream", PILLOW, ids=[n for n, _ in PILLOW])
def test_twin_pillow_streams(name, stream):
    assert np.array_equal(vb.webp_decode_host_twin(stream), pillow(stream)), name


@pytest.mark.parametrize("name,stream", WRITER, ids=[n for n, _ in WRITER])
def test_twin_writer_streams(name, stream):
    want = pillow_or_none(stream)
    assert want is not None, "libwebp refused the written stream " + name
    assert np.array_equal(vb.webp_decode_host_twin(stream), want), name


def test_fixture_and_icc():
    s = open(os.path.join(GOLDEN, "1.webp"), "rb").read()
    assert vb.webp_geometry(s) == (550, 368, 3)
    assert np.array_equal(vb.webp_decode_host_twin(s), pillow(s))
    assert vb.webp_icc_profile(s) is None
    prof = open(os.path.join(os.path.dirname(GOLDEN), "profiles", "sRGB.icm"), "rb").read()
    icc = pil_webp(content("photo", 45, 61, 3), quality=80, icc_profile=prof)
    assert icc[12:16] == b"VP8X"
    assert vb.webp_icc_profile(icc) == prof
    assert np.array_equal(vb.webp_decode_host_twin(icc), pillow(icc))


def _refusal(stream, match):
    with pytest.raises(vb.Error, match=match):
        vb.webp_decode_host_twin(stream)
    with pytest.raises(vb.Error, match=match):
        vb.webp_geometry(stream)


def test_refusals():
    a = content("photo", 20, 30, 1)
    _refusal(pil_webp(a, lossless=True), "lossless")
    rgba = np.dstack([a, np.full(a.shape[:2], 128, np.uint8)])
    _refusal(pil_webp(rgba, quality=80), "alpha")
    b = io.BytesIO()
    PIL.fromarray(a).save(b, "WEBP", save_all=True, append_images=[PIL.fromarray(a[::-1].copy())], quality=70)
    _refusal(b.getvalue(), "animated")
    _refusal(open(os.path.join(GOLDEN, "looks-like-svg.webp"), "rb").read(), "alpha|animated|lossless")
    _refusal(open(os.path.join(GOLDEN, "big-height.webp"), "rb").read(), "alpha|animated|lossless")
    s = pil_webp(a, quality=70)
    _refusal(s[:4] + struct.pack("<I", len(s)) + s[8:], "RIFF size")
    _refusal(s[:4] + struct.pack("<I", 8) + s[8:], "RIFF size")
    _refusal(b"RIFF" + s[4:8] + b"WEBQ" + s[12:], "signature")
    v = vp8_payload(s)
    _refusal(riff([(b"VP8 ", bytes([v[0] | 1]) + v[1:])]), "not a key frame")
    _refusal(riff([(b"VP8 ", v[:3] + b"\x9d\x01\x2b" + v[6:])]), "start code")


def _cut(stream, k):
    """the stream with its VP8 payload cut to k bytes, and the RIFF and chunk sizes made to agree"""
    return riff([(b"VP8 ", vp8_payload(stream)[:k])])


def truncation_streams():
    s1 = pil_webp(content("photo", 40, 50, 5), quality=90)
    return [("pillow", s1), ("parts4", vp8_stream(77, h=64, w=48, parts=4)), ("parts8", vp8_stream(78, h=50, w=33, parts=8))]


@pytest.mark.parametrize("name,stream", truncation_streams(), ids=[n for n, _ in truncation_streams()])
def test_truncation(name, stream):
    """cut inside every partition: the twin fails exactly where libwebp does, and otherwise decodes what it decodes"""
    n = len(vp8_payload(stream))
    points = sorted(set(list(range(10, min(n, 80))) + list(range(10, n, max(1, n // 150))) + list(range(max(10, n - 40), n))))
    fails = 0
    for k in points:
        c = _cut(stream, k)
        want = pillow_or_none(c)
        if want is None:
            fails += 1
            with pytest.raises(vb.Error):
                vb.webp_decode_host_twin(c)
        else:
            assert np.array_equal(vb.webp_decode_host_twin(c), want), (name, k)
    assert fails > 0


def test_abi():
    L = C.CDLL(vb.library_path())
    for name in ("vb200_webp_geometry", "vb200_webp_decode_batch", "vb200_webpload_buffer", "vb200_webp_icc_profile",
                 "vb200_debug_webp_decode", "vb200_debug_webp_tables"):
        assert hasattr(L, name), name
    s = PILLOW[3][1]
    h, w = pillow(s).shape[:2]
    assert vb.webp_decode_batch.__doc__ and vb.webp_geometry(s) == (w, h, 3)
    # geometry of a batch needs no device
    from libvips_b200 import _batch_geometry
    assert _batch_geometry(vb.lib().vb200_webp_decode_batch, [s, s]) == (w, h, 3)
    with pytest.raises(vb.Error, match="one geometry"):
        _batch_geometry(vb.lib().vb200_webp_decode_batch, [s, pil_webp(content("flat", h + 1, w, 0))])
    with pytest.raises(vb.Error, match="frame 1: lossless"):
        _batch_geometry(vb.lib().vb200_webp_decode_batch, [s, pil_webp(content("flat", h, w, 0), lossless=True)])
    # a thumbnail of a WebP stream is refused with the WebP reason, not a JPEG parse error
    out = vb.CImage()
    out.where = vb.HOST
    rc = vb.lib().vb200_thumbnail_buffer(s, len(s), C.byref(out), 32, 32, 0)
    msg = vb.lib().vb200_error_buffer().decode()
    vb.lib().vb200_error_clear()
    assert rc == -1 and "WebP shrink-on-load" in msg, msg


# ------------------------------------------------------------------ on the device


def all_cpu_streams():
    return [s for _, s in PILLOW] + [s for _, s in WRITER]


@pytest.mark.gpu
def test_gpu_every_stream(vb):
    by_geometry = {}
    for s in all_cpu_streams():
        by_geometry.setdefault(vb.webp_geometry(s), []).append(s)
    for g, streams in by_geometry.items():
        got = vb.webp_decode_batch(streams)
        for i, s in enumerate(streams):
            assert np.array_equal(got[i], vb.webp_decode_host_twin(s)), (g, i)


@pytest.mark.gpu
def test_gpu_thousands_of_small_frames(vb):
    streams = [vp8_stream(5000 + i % 97, h=24, w=20) for i in range(3000)]
    got = vb.webp_decode_batch(streams)
    twin = [vb.webp_decode_host_twin(streams[k]) for k in range(97)]
    for i in range(3000):
        assert np.array_equal(got[i], twin[i % 97]), i


@pytest.mark.gpu
def test_gpu_strides_and_chunks(vb):
    import torch
    streams = [vp8_stream(6000 + i, h=37, w=45) for i in range(9)] + [pil_webp(content("photo", 37, 45, i), quality=60) for i in range(5)]
    want = np.stack([vb.webp_decode_host_twin(s) for s in streams])
    assert np.array_equal(vb.webp_decode_batch(streams), want)
    h, w = 37, 45
    bpl, stride = w * 3 + 5, (w * 3 + 5) * h + 11
    dev = torch.full((stride * len(streams),), 77, dtype=torch.uint8, device="cuda")
    vb.webp_decode_batch(streams, out_ptr=dev.data_ptr(), out_bpl=bpl, out_frame_stride=stride)
    torch.cuda.synchronize()
    d = dev.cpu().numpy()
    for i in range(len(streams)):
        frame = d[i * stride:i * stride + bpl * h].reshape(h, bpl)
        assert np.array_equal(frame[:, :w * 3].reshape(h, w, 3), want[i]), i
        assert (frame[:, w * 3:] == 77).all()
    img = vb.Image.webpload_buffer(streams[0])
    assert np.array_equal(img.numpy(), want[0])
    assert vb.webp_times() is None
    os.environ["VB200_WEBP_TIMING"] = "1"
    try:
        assert np.array_equal(vb.webp_decode_batch(streams), want)
        t = vb.webp_times()
        assert set(t) == {"header", "tokens", "recon", "rgb"} and all(v > 0 for v in t.values()), t
    finally:
        del os.environ["VB200_WEBP_TIMING"]


def _decode_raw(streams, out, location, bpl, stride):
    b = vb.StreamBatch(streams)
    ww, hh, bb = C.c_int(), C.c_int(), C.c_int()
    rc = vb.lib().vb200_webp_decode_batch(b.ptrs, b.lens, b.n, C.c_void_p(out), location, bpl, stride, C.byref(ww), C.byref(hh), C.byref(bb))
    msg = vb.lib().vb200_error_buffer().decode()
    vb.lib().vb200_error_clear()
    return rc, msg


@pytest.mark.gpu
def test_gpu_chunks(vb):
    """a batch split by the device budget into chunks of 2-3 frames decodes as one, into host and device memory at padded
    strides, and a bad frame in a later chunk is named by its index in the whole batch"""
    import torch
    h, w = 37, 45
    streams = [vp8_stream(6100 + i, h=h, w=w, parts=1 + i % 4 // 2 * 3) for i in range(9)]
    streams += [pil_webp(content("photo", h, w, 20 + i), quality=40 + 10 * i) for i in range(5)]
    want = np.stack([vb.webp_decode_host_twin(s) for s in streams])
    n, bpl, stride = len(streams), w * 3 + 5, (w * 3 + 5) * h + 11
    L = vb.lib()
    try:
        L.vb200_debug_png_set_budget(40000)
        before = vb.launch_count()
        assert np.array_equal(vb.webp_decode_batch(streams), want)
        assert vb.launch_count() - before >= 4 * 5, "the batch did not split into chunks"
        host = np.full(stride * n, 77, np.uint8)
        rc, msg = _decode_raw(streams, host.ctypes.data, vb.HOST, bpl, stride)
        assert rc == 0, msg
        dev = torch.full((stride * n,), 77, dtype=torch.uint8, device="cuda")
        rc, msg = _decode_raw(streams, dev.data_ptr(), vb.DEVICE, bpl, stride)
        assert rc == 0, msg
        torch.cuda.synchronize()
        for d in (host, dev.cpu().numpy()):
            for i in range(n):
                frame = d[i * stride:i * stride + bpl * h].reshape(h, bpl)
                assert np.array_equal(frame[:, :w * 3].reshape(h, w, 3), want[i]), i
                assert (frame[:, w * 3:] == 77).all() and (d[i * stride + bpl * h:(i + 1) * stride] == 77).all(), i
        # a frame that fails while decoding, in a later chunk
        cut = next(c for c in (_cut(streams[2], k) for k in range(len(vp8_payload(streams[2])) - 1, 10, -1)) if pillow_or_none(c) is None)
        batch = streams[:11] + [cut] + streams[12:]
        host = np.full(stride * n, 0xA5, np.uint8)
        rc, msg = _decode_raw(batch, host.ctypes.data, vb.HOST, bpl, stride)
        assert rc == -1 and "frame 11:" in msg, msg
        assert (host == 0xA5).all()
        rc, msg = _decode_raw(batch, dev.data_ptr(), vb.DEVICE, bpl, stride)
        assert rc == -1 and "frame 11:" in msg, msg
        L.vb200_debug_png_set_budget(100)
        with pytest.raises(vb.Error, match="more than the 100 allowed"):
            vb.webp_decode_batch(streams[:2])
    finally:
        L.vb200_debug_png_set_budget(0)


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", [(17, 16383), (16383, 17), (4096, 4096)])
def test_gpu_large_frames(vb, h, w):
    s = vp8_stream(7000 + h, h=h, w=w, parts=8) if h * w < 4096 * 4096 else pil_webp(content("photo", h, w, 1), quality=85)
    assert np.array_equal(vb.webp_decode_batch([s])[0], vb.webp_decode_host_twin(s))


@pytest.mark.gpu
def test_gpu_two_threads(vb):
    streams = [vp8_stream(8000 + i, h=50, w=60) for i in range(40)]
    want = np.stack([vb.webp_decode_host_twin(s) for s in streams])
    res = [None, None]

    def run(k):
        vb.init(0)
        res[k] = all(np.array_equal(vb.webp_decode_batch(streams), want) for _ in range(3))

    th = [threading.Thread(target=run, args=(k,)) for k in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert res == [True, True]


@pytest.mark.gpu
def test_gpu_batch_or_nothing(vb):
    import torch
    streams = [vp8_stream(9000 + i, h=30, w=30, parts=2) for i in range(12)]
    cut = next(_cut(streams[5], k) for k in range(len(vp8_payload(streams[5])) - 1, 10, -1) if pillow_or_none(_cut(streams[5], k)) is None)
    batch = streams[:5] + [cut] + streams[6:]
    L = vb.lib()
    pool = L.vb200_debug_dz_pool_used()
    out = np.full((len(batch), 30, 30, 3), 0xA5, np.uint8)
    b = vb.StreamBatch(batch)
    ww, hh, bb = C.c_int(), C.c_int(), C.c_int()
    rc = L.vb200_webp_decode_batch(b.ptrs, b.lens, b.n, out.ctypes.data_as(C.c_void_p), vb.HOST, 90, 2700, C.byref(ww), C.byref(hh), C.byref(bb))
    msg = L.vb200_error_buffer().decode()
    L.vb200_error_clear()
    assert rc == -1 and "frame 5:" in msg, msg
    assert (out == 0xA5).all()
    dev = torch.full((out.size,), 0xA5, dtype=torch.uint8, device="cuda")
    assert L.vb200_webp_decode_batch(b.ptrs, b.lens, b.n, C.c_void_p(dev.data_ptr()), vb.DEVICE, 90, 2700, None, None, None) == -1
    L.vb200_error_clear()
    torch.cuda.synchronize()
    assert (dev.cpu().numpy() == 0xA5).all()
    assert L.vb200_debug_dz_pool_used() == pool
    vb.webp_decode_batch(streams)
    assert L.vb200_debug_dz_pool_used() == pool


@pytest.mark.gpu
def test_gpu_frames_feed_a_device_op(vb):
    """a decoded frame used in place by dzsave equals dzsave of the twin's pixels"""
    import torch
    s = pil_webp(content("photo", 300, 410, 2), quality=80)
    frame = torch.empty((300, 410, 3), dtype=torch.uint8, device="cuda")
    vb.webp_decode_batch([s], out_ptr=frame.data_ptr())
    got = vb.dzsave(None, "w", in_ptr=frame.data_ptr(), shape=(300, 410, 3))
    want = vb.dzsave_host_twin(vb.webp_decode_host_twin(s), "w")
    assert [t.bytes for t in got.tiles] == [t.bytes for t in want.tiles]

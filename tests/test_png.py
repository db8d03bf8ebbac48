"""PNG decode (csrc/png.cu): vips_pngload_buffer as spngload.c gives it, on the device and through its host twin.

The CPU half pins the host twin (the same per-symbol, per-byte and per-pixel code the kernels run) to a PNG writer of this
file's own, to Pillow's decoder and, for the inflate alone, to Python's zlib: where zlib's raw inflate refuses a deflate
stream the twin refuses it, and where zlib accepts one the twin gives its bytes.  The GPU half pins the batch decoder and the
thumbnail entry points to the host twin, Pillow and the oracle."""
import ctypes as C
import io
import os
import struct
import zlib

import numpy as np
import pytest
from PIL import Image as PIL

import libvips_b200 as vb

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "png")


# ---------------------------------------------------------------------------------------------------------- the writer

def chunk(kind, data, bad_crc=False):
    crc = zlib.crc32(kind + data) ^ (0x5A5A5A5A if bad_crc else 0)
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", crc & 0xFFFFFFFF)


def pack_rows(samples, depth):
    """[h][w * spp] samples -> [h][rowbytes], MSB first below 8 bits"""
    if depth == 8:
        return samples.astype(np.uint8)
    per = 8 // depth
    h, n = samples.shape
    padded = np.zeros((h, -(-n // per) * per), np.uint8)
    padded[:, :n] = samples
    g = padded.reshape(h, -1, per).astype(np.uint16)
    out = np.zeros(g.shape[:2], np.uint16)
    for k in range(per):
        out |= g[:, :, k] << (8 - depth * (k + 1))
    return out.astype(np.uint8)


def filter_rows(rows, bpp, filters):
    """PNG 2nd edition 9: each row filtered with its own type; -> bytes with the filter byte per row"""
    h, rb = rows.shape
    r = rows.astype(np.int32)
    out = bytearray()
    for y in range(h):
        ft = int(filters[y])
        cur = r[y]
        up = r[y - 1] if y else np.zeros(rb, np.int32)
        left = np.concatenate([np.zeros(bpp, np.int32), cur[:-bpp]]) if rb > bpp else np.zeros(rb, np.int32)
        ul = np.concatenate([np.zeros(bpp, np.int32), up[:-bpp]]) if rb > bpp else np.zeros(rb, np.int32)
        if ft == 0:
            f = cur
        elif ft == 1:
            f = cur - left
        elif ft == 2:
            f = cur - up
        elif ft == 3:
            f = cur - (left + up) // 2
        else:
            p = left + up - ul
            pa, pb, pc = abs(p - left), abs(p - up), abs(p - ul)
            pred = np.where((pa <= pb) & (pa <= pc), left, np.where(pb <= pc, up, ul))
            f = cur - pred
        out.append(ft)
        out += (f & 255).astype(np.uint8).tobytes()
    return bytes(out)


def write_png(samples, ct, depth, palette=None, trns=None, filters=None, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, wbits=15,
              flush=None, idat_sizes=None, empty_idat=False, before=(), after=(), bad_crc=False, bad_adler=False, raw_z=None):
    """samples: [h][w][spp] ints.  filters: one type per row (default: cycling 0..4).  flush: Z_SYNC_FLUSH / Z_FULL_FLUSH after
    the first half of the scanlines.  idat_sizes: IDAT payload sizes (the rest in the last one).  raw_z: the zlib stream to
    use instead."""
    h, w = samples.shape[:2]
    spp = samples.shape[2]
    rows = pack_rows(samples.reshape(h, w * spp), depth)
    bpp = max(1, spp * depth // 8)
    if filters is None:
        filters = [y % 5 for y in range(h)]
    scan = filter_rows(rows, bpp, filters)
    if raw_z is None:
        co = zlib.compressobj(level, zlib.DEFLATED, wbits, 9, strategy)
        if flush is not None:
            z = co.compress(scan[:len(scan) // 2]) + co.flush(flush) + co.compress(scan[len(scan) // 2:]) + co.flush()
        else:
            z = co.compress(scan) + co.flush()
    else:
        z = raw_z
    if bad_adler:
        z = z[:-4] + bytes(b ^ 0xFF for b in z[-4:])
    out = b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, ct, 0, 0, 0), bad_crc)
    out += b"".join(before)
    if palette is not None:
        out += chunk(b"PLTE", np.asarray(palette, np.uint8).tobytes(), bad_crc)
    if trns is not None:
        out += chunk(b"tRNS", trns, bad_crc)
    parts = []
    rest = z
    for n in idat_sizes or ():
        parts.append(rest[:n])
        rest = rest[n:]
    parts.append(rest)
    if empty_idat:
        parts.insert(1, b"")
    out += b"".join(chunk(b"IDAT", p, bad_crc) for p in parts)
    out += b"".join(after)
    return out + chunk(b"IEND", b"", bad_crc)


def expected(samples, ct, depth, palette=None, trns=None):
    """spngload.c's output for the writer's samples"""
    s = samples.astype(np.int64)
    if ct == 3:
        pal = np.zeros((256, 4), np.uint8)
        pal[:, 3] = 255
        pal[:len(palette), :3] = palette
        if trns is not None:
            pal[:len(trns), 3] = np.frombuffer(trns, np.uint8)
        return pal[s[:, :, 0]][:, :, :4 if trns is not None else 3]
    if ct == 0:
        g = (s[:, :, 0] * (255 // ((1 << depth) - 1))).astype(np.uint8)
        if trns is None:
            return g[:, :, None]
        key = struct.unpack(">H", trns)[0]
        return np.stack([g, np.where(s[:, :, 0] == key, 0, 255).astype(np.uint8)], 2)
    if ct == 2 and trns is not None:
        key = np.array(struct.unpack(">HHH", trns))
        a = np.where((s == key).all(2), 0, 255).astype(np.uint8)
        return np.concatenate([samples.astype(np.uint8), a[:, :, None]], 2)
    return samples.astype(np.uint8)


def pillow(stream, bands):
    """Pillow's decode in spngload's layout"""
    im = PIL.open(io.BytesIO(stream))
    im.load()
    if im.mode == "P":
        return np.array(im.convert("RGBA" if bands == 4 else "RGB"))
    if im.mode in ("1", "L"):
        g = np.array(im.convert("L"))
        if bands == 2:
            return np.stack([g, np.where(g == im.info["transparency"], 0, 255).astype(np.uint8)], 2)
        return g[:, :, None]
    if im.mode == "RGB" and bands == 4:
        a = np.array(im)
        key = np.array(im.info["transparency"])
        return np.concatenate([a, np.where((a == key).all(2), 0, 255).astype(np.uint8)[:, :, None]], 2)
    a = np.array(im)
    return a if a.ndim == 3 else a[:, :, None]


# every in-scope kind: (name, ct, depth, spp, palette entries, tRNS kind)
KINDS = [("grey8", 0, 8, 1, 0, None), ("grey4", 0, 4, 1, 0, None), ("grey2", 0, 2, 1, 0, None), ("grey1", 0, 1, 1, 0, None),
         ("grey8_trns", 0, 8, 1, 0, "key"), ("ga8", 4, 8, 2, 0, None), ("rgb8", 2, 8, 3, 0, None), ("rgb8_trns", 2, 8, 3, 0, "key"),
         ("rgba8", 6, 8, 4, 0, None), ("pal8", 3, 8, 1, 200, None), ("pal4", 3, 4, 1, 16, None), ("pal2", 3, 2, 1, 3, None),
         ("pal1", 3, 1, 1, 2, None), ("pal8_trns", 3, 8, 1, 200, "alpha"), ("pal4_trns", 3, 4, 1, 11, "alpha"),
         ("pal1_trns", 3, 1, 1, 2, "alpha")]


def make(kind, h, w, seed, **kw):
    """(stream, expected pixels) of one kind at h x w"""
    name, ct, depth, spp, npal, tk = kind
    rng = np.random.default_rng(seed)
    top = npal if ct == 3 else 1 << depth
    s = rng.integers(0, top, (h, w, spp))
    if depth == 8 and ct != 3:  # runs and repeats, so that matches happen
        s[:, : w // 2] = s[:, :1]
    palette = rng.integers(0, 256, (npal, 3)) if ct == 3 else None
    trns = None
    if tk == "key":
        key = [int(v) for v in s[0, 0]]
        trns = struct.pack(">" + "H" * len(key), *key)
    elif tk == "alpha":
        trns = rng.integers(0, 256, max(1, npal - 1), dtype=np.uint8).tobytes()
    return write_png(s, ct, depth, palette, trns, **kw), expected(s, ct, depth, palette, trns)


SIZES = [(1, 1), (1, 13), (13, 1), (7, 9), (5, 33), (3, 127), (17, 64)]


@pytest.mark.parametrize("kind", KINDS, ids=[k[0] for k in KINDS])
def test_host_twin_every_kind_and_size(kind):
    for i, (h, w) in enumerate(SIZES):
        stream, want = make(kind, h, w, seed=i)
        got = vb.png_decode_host_twin(stream)
        assert got.shape == want.shape, (kind[0], h, w)
        assert np.array_equal(got, want), (kind[0], h, w)
        assert np.array_equal(got, pillow(stream, want.shape[2])), (kind[0], h, w)


WRITER_VARIANTS = [dict(level=0), dict(level=1), dict(level=6), dict(level=9), dict(strategy=zlib.Z_FILTERED),
                   dict(strategy=zlib.Z_HUFFMAN_ONLY), dict(strategy=zlib.Z_RLE), dict(strategy=zlib.Z_FIXED)] + \
                  [dict(wbits=b) for b in range(9, 16)] + \
                  [dict(flush=zlib.Z_SYNC_FLUSH), dict(flush=zlib.Z_FULL_FLUSH), dict(idat_sizes=[1] * 40, empty_idat=True),
                   dict(filters="zero"), dict(filters="sub"), dict(filters="up"), dict(filters="avg"), dict(filters="paeth")]
ANCILLARY = [chunk(b"tEXt", b"Comment\0hello"), chunk(b"zTXt", b"Title\0\0" + zlib.compress(b"a title")), chunk(b"gAMA", struct.pack(">I", 45455)),
             chunk(b"pHYs", struct.pack(">IIB", 2835, 2835, 1)), chunk(b"prVt", b"private data")]


def _variant(v, h):
    v = dict(v)
    if isinstance(v.get("filters"), str):
        v["filters"] = [["zero", "sub", "up", "avg", "paeth"].index(v["filters"])] * h
    return v


@pytest.mark.parametrize("vi", range(len(WRITER_VARIANTS)))
def test_host_twin_writer_variants(vi):
    for kind in KINDS:
        for h, w in ((9, 31), (40, 25)):
            stream, want = make(kind, h, w, seed=vi, **_variant(WRITER_VARIANTS[vi], h))
            got = vb.png_decode_host_twin(stream)
            assert np.array_equal(got, want), (kind[0], WRITER_VARIANTS[vi])
            assert np.array_equal(got, pillow(stream, want.shape[2])), (kind[0], WRITER_VARIANTS[vi])


def test_host_twin_ancillary_chunks_and_bad_checksums():
    icc = zlib.compress(bytes(range(256)) * 3)
    iccp = chunk(b"iCCP", b"profile\0\0" + icc)
    for kind in KINDS:
        stream, want = make(kind, 11, 19, seed=3, before=[iccp] + ANCILLARY, after=ANCILLARY)
        assert np.array_equal(vb.png_decode_host_twin(stream), want), kind[0]
        assert np.array_equal(pillow(stream, want.shape[2]), want), kind[0]
        # CRCs and the Adler-32 are not checked (spngload.c:346-352)
        for kw in (dict(bad_crc=True), dict(bad_adler=True), dict(bad_crc=True, bad_adler=True)):
            stream, want = make(kind, 11, 19, seed=3, before=ANCILLARY, **kw)
            assert np.array_equal(vb.png_decode_host_twin(stream), want), (kind[0], kw)


def test_long_matches_and_far_distances():
    """matches of length 258 at distance 32 768, and every distance up to it"""
    rng = np.random.default_rng(5)
    block = rng.integers(0, 256, (1, 32767, 1))
    s = np.concatenate([block, block, block], 1).reshape(3, 32767, 1)
    stream = write_png(s, 0, 8, filters=[0, 0, 0], level=9)
    assert np.array_equal(vb.png_decode_host_twin(stream), s.astype(np.uint8))
    raw = bytes(rng.integers(0, 256, 32768, dtype=np.uint8)) * 4 + b"\0" * 1000
    z = zlib.compress(raw, 9)[2:-4]
    assert vb.inflate_host_twin(z, len(raw)) == raw


PIL_MODES = [("L", {}), ("LA", {}), ("RGB", {}), ("RGBA", {}), ("P", {"bits": 1}), ("P", {"bits": 2}), ("P", {"bits": 4}), ("P", {}),
             ("1", {}), ("L", {"transparency": 7}), ("RGB", {"transparency": (1, 2, 3)}), ("P", {"transparency": 0}),
             ("P", {"bits": 4, "transparency": 3})]


@pytest.mark.parametrize("mi", range(len(PIL_MODES)))
def test_pillow_written(mi):
    mode, kw = PIL_MODES[mi]
    rng = np.random.default_rng(mi)
    for h, w in ((1, 1), (23, 37)):
        if mode in ("P", "1"):
            ncol = 1 << kw.get("bits", 8) if mode == "P" else 2
            a = rng.integers(0, ncol, (h, w), dtype=np.uint8)
            im = PIL.fromarray(a * (255 if mode == "1" else 1), "L").convert("1") if mode == "1" else PIL.fromarray(a, "P")
            if mode == "P":
                im.putpalette(list(rng.integers(0, 256, 3 * ncol, dtype=np.uint8)))
        else:
            nb = {"L": 1, "LA": 2, "RGB": 3, "RGBA": 4}[mode]
            a = rng.integers(0, 256, (h, w, nb), dtype=np.uint8)
            a[: h // 2, : w // 2] = [1, 2, 3, 4][:nb] if "transparency" in kw else a[: h // 2, : w // 2]
            if "transparency" in kw and mode == "L":
                a[0, 0] = 7
            im = PIL.fromarray(a[:, :, 0] if nb == 1 else a, mode)
        for level in list(range(10)) + ["optimize"]:
            b = io.BytesIO()
            opts = dict(kw)
            if level == "optimize":
                opts["optimize"] = True
            else:
                opts["compress_level"] = level
            im.save(b, "PNG", **opts)
            s = b.getvalue()
            got = vb.png_decode_host_twin(s)
            assert np.array_equal(got, pillow(s, got.shape[2])), (mode, kw, level)


def test_reference_known_answers():
    with open(os.path.join(GOLDEN, "indexed.png"), "rb") as f:
        a = vb.png_decode_host_twin(f.read())
    assert a.shape == (442, 290, 3)
    assert list(a[10, 10]) == [148, 131, 109]
    # the 1-bit round trip pins 1 -> 255 (test_foreign.py:631-635)
    s = write_png(np.array([[[0], [1], [1], [0], [1]]]), 0, 1)
    assert list(vb.png_decode_host_twin(s)[0, :, 0]) == [0, 255, 255, 0, 255]
    for name in ("indexed", "rgba", "trans-x", "cogs"):
        with open(os.path.join(GOLDEN, name + ".png"), "rb") as f:
            s = f.read()
        got = vb.png_decode_host_twin(s)
        assert np.array_equal(got, pillow(s, got.shape[2])), name


# ---------------------------------------------------------------------------------------------------------- the acceptance rule

class Bits:
    """an LSB-first bit writer for hand-made deflate streams"""

    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, value, n):
        self.v |= (value & ((1 << n) - 1)) << self.n
        self.n += n

    def code(self, code, n):  # Huffman codes go MSB first
        self.put(int(format(code, "0%db" % n)[::-1], 2) if n else 0, n)

    def bytes(self):
        return self.v.to_bytes((self.n + 7) // 8, "little")


def canonical(lengths):
    """RFC 1951 3.2.2: the codes of a set of lengths"""
    bl = [0] * 16
    for ln in lengths:
        if ln:
            bl[ln] += 1
    code, nxt = 0, [0] * 16
    for b in range(1, 16):
        code = (code + bl[b - 1]) << 1
        nxt[b] = code
    out = []
    for ln in lengths:
        out.append(nxt[ln] if ln else None)
        if ln:
            nxt[ln] += 1
    return out


def fixed_lit(b, sym):
    if sym < 144:
        b.code(0x30 + sym, 8)
    elif sym < 256:
        b.code(0x190 + sym - 144, 9)
    elif sym < 280:
        b.code(sym - 256, 7)
    else:
        b.code(0xC0 + sym - 280, 8)


ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
CL_OK = [4] * 13 + [5] * 6  # a complete code-length code (13 / 16 + 6 / 32 = 1)
LIT_OK = [8] * 226 + [9] * 60  # 286 symbols, complete
DIST_OK = [5] * 28 + [4] * 2  # 30 symbols, complete


def dynamic(symbols, lit=LIT_OK, dist=DIST_OK, cl=CL_OK, hlit=None, hdist=None, cl_symbols=None, final=1):
    """a dynamic block: header, code lengths sent one symbol each (or cl_symbols: (sym, extra bits, n) triples), then symbols:
    ints for literals / end-of-block, (length symbol, extra, distance symbol, extra) for matches"""
    b = Bits()
    b.put(final, 1)
    b.put(2, 2)
    b.put((len(lit) - 257) if hlit is None else hlit, 5)
    b.put((len(dist) - 1) if hdist is None else hdist, 5)
    b.put(15, 4)
    cl_by_sym = dict(zip(ORDER, cl))
    for s in ORDER:
        b.put(cl_by_sym[s], 3)
    clc = canonical([cl_by_sym.get(i, 0) for i in range(19)])
    cll = [cl_by_sym.get(i, 0) for i in range(19)]
    for s, extra, n in cl_symbols or [(ln, 0, 0) for ln in list(lit) + list(dist)]:
        b.code(clc[s], cll[s])
        if n:
            b.put(extra, n)
    lc, dc = canonical(lit), canonical(dist)
    for s in symbols:
        if isinstance(s, tuple):
            ls, le, ds, de = s
            b.code(lc[ls], lit[ls])
            b.put(*le)
            b.code(dc[ds], dist[ds])
            b.put(*de)
        else:
            b.code(lc[s], lit[s])
    return b.bytes()


def fixed(symbols, final=1):
    b = Bits()
    b.put(final, 1)
    b.put(1, 2)
    for s in symbols:
        if isinstance(s, tuple):
            ls, le, ds, de = s
            fixed_lit(b, ls)
            b.put(*le)
            b.code(ds, 5)
            b.put(*de)
        else:
            fixed_lit(b, s)
    return b.bytes()


def zlib_verdict(raw):
    """Python's zlib on raw deflate data: the bytes, or None where it refuses (an error, or the stream does not end)"""
    d = zlib.decompressobj(-15)
    try:
        out = d.decompress(raw)
    except zlib.error:
        return None
    return out if d.eof else None


def twin_verdict(raw):
    try:
        return vb.inflate_host_twin(raw, 1 << 22)
    except vb.Error:
        return None


def hand_made():
    lit1 = [0] * 286
    lit1[65] = lit1[256] = 1  # 'A' and end-of-block only
    one_dist = [1] + [0] * 29  # a single distance code of length 1: incomplete, allowed
    over = [8] * 227 + [9] * 59
    under = [8] * 225 + [9] * 61
    no_eob = list(LIT_OK)
    no_eob[256] = 0
    return {
        "fixed ok": fixed([65, 66, (257, (0, 0), 0, (0, 0)), 256]),
        "fixed lit 286": fixed([65, 286, 256]),
        "fixed lit 287": fixed([65, 287, 256]),
        "fixed dist 30": fixed([65, 66, (257, (0, 0), 30, (0, 0)), 256]),
        "fixed dist 31": fixed([65, 66, (257, (0, 0), 31, (0, 0)), 256]),
        "distance before the start": fixed([65, (257, (0, 0), 1, (0, 0)), 256]),
        "distance at the start": fixed([65, 66, (257, (0, 0), 1, (0, 0)), 256]),
        "length 258 distance 1": fixed([65, (285, (0, 0), 0, (0, 0)), 256]),
        "dynamic ok": dynamic([65, 66, 67, (257, (0, 0), 2, (0, 0)), 256]),
        "dynamic literals only, no distances": dynamic([65, 256], lit=lit1, dist=[0]),
        "dynamic match without distances": dynamic([65, (257, (0, 0), 0, (0, 0)), 256], lit=[1] * 2 + [0] * 255 + [1, 1] + [0] * 27, dist=[0]),
        "dynamic one distance code": dynamic([65, 66, (257, (0, 0), 0, (0, 0)), 256], lit=LIT_OK, dist=one_dist),
        "dynamic lit over-subscribed": dynamic([65, 256], lit=over),
        "dynamic lit incomplete": dynamic([65, 256], lit=under),
        "dynamic dist over-subscribed": dynamic([65, 256], dist=[4] * 30),
        "dynamic dist incomplete": dynamic([65, 256], dist=[5] * 30),
        "code-length code over-subscribed": dynamic([65, 256], cl=[4] * 19),
        "code-length code incomplete": dynamic([65, 256], cl=[5] * 19),
        "code-length code empty": dynamic([65, 256], cl=[0] * 19),
        "HLIT 287": dynamic([65, 256], lit=LIT_OK + [0]),
        "HLIT 288": dynamic([65, 256], lit=LIT_OK + [0, 0]),
        "HDIST 31": dynamic([65, 256], dist=DIST_OK + [0]),
        "HDIST 32": dynamic([65, 256], dist=DIST_OK + [0, 0]),
        "no end-of-block code": dynamic([65], lit=no_eob),
        "repeat with nothing before": dynamic([65, 256], cl_symbols=[(16, 0, 2)] + [(ln, 0, 0) for ln in LIT_OK + DIST_OK][3:]),
        "repeat past the end": dynamic([65, 256], cl_symbols=[(ln, 0, 0) for ln in LIT_OK + DIST_OK][:-2] + [(18, 0, 7)]),
        "stored ok": b"\x01\x03\x00\xfc\xffabc",
        "stored bad NLEN": b"\x01\x03\x00\xfc\xfeabc",
        "stored short": b"\x01\x03\x00\xfc\xffab",
        "stored empty then fixed": b"\x00\x00\x00\xff\xff" + fixed([65, 256]),
        "block type 3": b"\x07\x00",
        "empty": b"",
    }


def test_acceptance_rule_hand_made():
    for name, raw in hand_made().items():
        want = zlib_verdict(raw)
        got = twin_verdict(raw)
        assert (got is None) == (want is None), (name, want, got)
        assert got == want, name
    # both sides of the rule are exercised
    v = {k: zlib_verdict(r) is not None for k, r in hand_made().items()}
    assert v["fixed ok"] and v["dynamic one distance code"] and not v["fixed lit 286"] and not v["dynamic lit incomplete"]


def test_acceptance_rule_mutants():
    rng = np.random.default_rng(7)
    data = bytes(rng.integers(0, 4, 3000, dtype=np.uint8)) + b"abcabcabd" * 50 + bytes(rng.integers(0, 256, 300, dtype=np.uint8))
    bases = [zlib.compressobj(lv, zlib.DEFLATED, -15, 9, st) for lv in (1, 6, 9) for st in (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FIXED, zlib.Z_HUFFMAN_ONLY)]
    streams = [c.compress(data) + c.flush() for c in bases] + list(hand_made().values())
    accepted = refused = 0
    for raw in streams:
        cuts = sorted(set(int(k) for k in np.linspace(0, len(raw), 25)))
        mutants = [raw[:k] for k in cuts]
        for _ in range(60):
            m = bytearray(raw)
            if not m:
                break
            for _ in range(int(rng.integers(1, 4))):
                i = int(rng.integers(0, len(m)))
                m[i] ^= 1 << int(rng.integers(0, 8))
            mutants.append(bytes(m))
        for m in mutants:
            want, got = zlib_verdict(m), twin_verdict(m)
            assert got == want, (raw[:16], m[:16])
            accepted += want is not None
            refused += want is None
    assert accepted > 50 and refused > 500


# ---------------------------------------------------------------------------------------------------------- declines and ICC

def _png_with_ihdr(depth, ct, interlace=0):
    return b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", 4, 4, depth, ct, 0, 0, interlace)) + \
        chunk(b"IDAT", zlib.compress(b"\0" * 80)) + chunk(b"IEND", b"")


def declined_streams():
    s = np.zeros((4, 4, 1), np.int64)
    good = write_png(s, 0, 8)
    pal = write_png(np.full((4, 4, 1), 3), 3, 8, palette=[[1, 2, 3]] * 3)
    idats = write_png(s, 0, 8, idat_sizes=[3])
    i2 = idats.index(b"IDAT", idats.index(b"IDAT") + 1) - 4
    split = idats[:i2] + chunk(b"tEXt", b"a\0b") + idats[i2:]
    z = zlib.compress(b"\0" * 20)
    return {
        "16-bit PNG not supported": open(os.path.join(GOLDEN, "sample.png"), "rb").read(),
        "Adam7-interlaced PNG not supported": write_png(s, 0, 8)[:8] + chunk(b"IHDR", struct.pack(">IIBBBBB", 4, 4, 8, 0, 0, 0, 1)) +
        write_png(s, 0, 8)[33:],
        "low-bit grey with tRNS not supported": write_png(np.zeros((4, 4, 1), np.int64), 0, 4, trns=b"\0\1"),
        "palette image without PLTE": write_png(np.zeros((4, 4, 1), np.int64), 3, 8),
        "bad PLTE chunk": write_png(np.zeros((4, 4, 1), np.int64), 3, 8, palette=np.zeros((0, 3))),
        "palette index beyond PLTE": pal,
        "IDAT chunks are not consecutive": split,
        "preset dictionary": write_png(s, 0, 8, raw_z=bytes([0x78, 0xBB]) + b"\0\0\0\0" + z[2:]),
        "not deflate": write_png(s, 0, 8, raw_z=bytes([0x79, (31 - 0x79 * 256 % 31) % 31]) + z[2:]),
        "bad FCHECK": write_png(s, 0, 8, raw_z=bytes([0x78, 0x9D]) + zlib.compress(b"\0" * 20)[2:]),
        "corrupt deflate stream": write_png(s, 0, 8, raw_z=zlib.compress(b"\0" * 20)[:2] + b"\x07\x00"),
        "inflates to fewer": write_png(s, 0, 8, raw_z=zlib.compress(b"\0" * 19)),
        "inflates to more": write_png(s, 0, 8, raw_z=zlib.compress(b"\0" * 21)),
        "frames over 2^28 pixels": good[:8] + chunk(b"IHDR", struct.pack(">IIBBBBB", 1 << 15, (1 << 13) + 1, 8, 0, 0, 0, 0)) + good[33:],
        "bad PNG filter type": write_png(s, 0, 8, raw_z=zlib.compress(b"\0\0\0\0\0" + b"\5\0\0\0\0" + b"\0" * 10)),
        "not a PNG stream": b"GIF89a" + good[6:],
    }


@pytest.mark.parametrize("reason", list(declined_streams()))
def test_declined(reason):
    s = declined_streams()[reason]
    with pytest.raises(vb.Error, match=reason.replace("^", r"\^")):
        vb.png_decode_host_twin(s)


def test_icc_profile():
    prof = bytes(range(256)) * 7 + b"end of profile"
    a = np.random.default_rng(3).integers(0, 256, (9, 11, 3), dtype=np.uint8)
    b = io.BytesIO()
    PIL.fromarray(a).save(b, "PNG", icc_profile=prof)
    s = b.getvalue()
    assert PIL.open(io.BytesIO(s)).info["icc_profile"] == prof
    assert vb.png_icc_profile(s) == prof
    b = io.BytesIO()
    PIL.fromarray(a).save(b, "PNG")
    assert vb.png_icc_profile(b.getvalue()) is None
    with open(os.path.join(GOLDEN, "indexed.png"), "rb") as f:
        assert vb.png_icc_profile(f.read()) is None


def test_geometry_without_a_device():
    streams = [make(KINDS[6], 5, 7, seed=i)[0] for i in range(3)] + [make(KINDS[9], 5, 7, seed=9)[0]]
    assert vb.png_geometry(streams) == (7, 5, 3)
    with pytest.raises(vb.Error, match="one geometry"):
        vb.png_geometry(streams + [make(KINDS[8], 5, 7, seed=1)[0]])
    with pytest.raises(vb.Error, match="frame 1: 16-bit"):
        vb.png_geometry([streams[0], declined_streams()["16-bit PNG not supported"]])


def test_abi_names():
    L = C.CDLL(vb.library_path())
    for name in ("vb200_png_decode_batch", "vb200_pngload_buffer", "vb200_png_icc_profile", "vb200_thumbnail_plan_run_png",
                 "vb200_debug_png_decode", "vb200_debug_inflate", "vb200_debug_png_set_budget"):
        assert hasattr(L, name), name
    assert vb.JpegBatch is vb.StreamBatch


# ---------------------------------------------------------------------------------------------------------- on the device

BY_BANDS = {1: ["grey8", "grey4", "grey2", "grey1"], 2: ["ga8", "grey8_trns"], 3: ["rgb8", "pal8", "pal4", "pal2", "pal1"],
            4: ["rgba8", "rgb8_trns", "pal8_trns", "pal4_trns", "pal1_trns"]}
KIND = {k[0]: k for k in KINDS}


def mixed_batch(bands, h, w):
    """every kind of one band count under every writer variant"""
    streams, want = [], []
    for vi, v in enumerate(WRITER_VARIANTS):
        for name in BY_BANDS[bands]:
            s, e = make(KIND[name], h, w, seed=vi * 31 + len(streams), **_variant(v, h))
            streams.append(s)
            want.append(e)
    return streams, np.stack(want)


def _sentinel_decode(streams, shape, location, ptr=None):
    b = vb.StreamBatch(streams)
    n, h, w, bands = shape
    ww, hh, bb = C.c_int(), C.c_int(), C.c_int()
    return vb.lib().vb200_png_decode_batch(b.ptrs, b.lens, b.n, C.c_void_p(ptr), location, w * bands, w * h * bands, C.byref(ww),
                                           C.byref(hh), C.byref(bb))


@pytest.mark.gpu
@pytest.mark.parametrize("bands", [1, 2, 3, 4])
def test_gpu_mixed_batches(vb, bands):
    import torch
    for h, w in ((1, 1), (37, 53), (70, 129)):
        streams, want = mixed_batch(bands, h, w)
        got = vb.png_decode_batch(streams)
        assert np.array_equal(got, want), (bands, h, w)
        for i in (0, len(streams) // 2, len(streams) - 1):
            assert np.array_equal(got[i], vb.png_decode_host_twin(streams[i]))
            assert np.array_equal(got[i], pillow(streams[i], bands))
        # into a device pointer, rows at an odd stride
        bpl = w * bands + 3
        stride = bpl * h + 5
        dev = torch.full((stride * len(streams),), 77, dtype=torch.uint8, device="cuda")
        vb.png_decode_batch(streams, out_ptr=dev.data_ptr(), out_bpl=bpl, out_frame_stride=stride)
        torch.cuda.synchronize()
        d = dev.cpu().numpy()
        for i in range(len(streams)):
            frame = d[i * stride:i * stride + bpl * h].reshape(h, bpl)
            assert np.array_equal(frame[:, :w * bands].reshape(h, w, bands), want[i]), (bands, h, w, i)
            assert (frame[:, w * bands:] == 77).all()


@pytest.mark.gpu
def test_gpu_fixtures_and_load_buffer(vb):
    for name in ("indexed", "rgba", "trans-x", "cogs"):
        with open(os.path.join(GOLDEN, name + ".png"), "rb") as f:
            s = f.read()
        want = vb.png_decode_host_twin(s)
        assert np.array_equal(vb.png_decode_batch([s, s])[1], want), name
        out = vb.CImage()
        out.where = vb.HOST
        vb._check(vb.lib().vb200_pngload_buffer(s, len(s), C.byref(out)))
        a = np.frombuffer(C.string_at(out.data, out.Ysize * out.bpl), np.uint8).reshape(out.Ysize, out.bpl)[:, :out.Xsize * out.Bands]
        assert np.array_equal(a.reshape(want.shape), want), name
        vb.lib().vb200_image_free(C.byref(out))
    assert list(vb.png_decode_batch([open(os.path.join(GOLDEN, "indexed.png"), "rb").read()])[0, 10, 10]) == [148, 131, 109]


@pytest.mark.gpu
def test_gpu_grid_limits(vb):
    ones = [make(KIND[k], 1, 1, seed=i)[0] for i, k in enumerate(["rgba8", "rgb8_trns", "pal4_trns", "pal8_trns"])]
    streams = [ones[i % 4] for i in range(70001)]
    got = vb.png_decode_batch(streams)
    for i in (0, 1, 2, 3, 65535, 65536, 70000):
        assert np.array_equal(got[i], vb.png_decode_host_twin(streams[i])), i
    for kind in ("rgb8", "pal2", "grey8"):
        s, want = make(KIND[kind], 70001, 3, seed=4)
        assert np.array_equal(vb.png_decode_batch([s])[0], want), kind


@pytest.mark.gpu
@pytest.mark.parametrize("bad", ["corrupt", "fewer", "more", "filter", "palette", "declined"])
def test_gpu_batch_or_nothing(vb, bad):
    import torch
    streams, want = mixed_batch(4, 9, 14)
    s0 = np.zeros((9, 14, 4), np.int64)
    z = zlib.compress(b"\0" * (9 * 57))
    bad_stream = {
        "corrupt": write_png(s0, 6, 8, raw_z=z[:2] + b"\x07" + z[3:]),
        "fewer": write_png(s0, 6, 8, raw_z=zlib.compress(b"\0" * (9 * 57 - 1))),
        "more": write_png(s0, 6, 8, raw_z=zlib.compress(b"\0" * (9 * 57 + 1))),
        "filter": write_png(s0, 6, 8, raw_z=zlib.compress(b"\0" * 57 * 4 + b"\7" + b"\0" * (57 * 5 - 1))),
        "palette": write_png(np.full((9, 14, 1), 5), 3, 8, palette=[[0, 0, 0]] * 5, trns=b"\0"),
        "declined": write_png(np.zeros((9, 14, 1), np.int64), 3, 8, palette=[[0, 0, 0]] * 2, trns=b"\0\0\0"),
    }[bad]
    k = 7
    batch = streams[:k] + [bad_stream] + streams[k:]
    L = vb.lib()
    pool = L.vb200_debug_dz_pool_used()
    shape = (len(batch), 9, 14, 4)
    out = np.full(shape, 0xA5, np.uint8)
    rc = _sentinel_decode(batch, shape, vb.HOST, out.ctypes.data)
    msg = L.vb200_error_buffer().decode()
    L.vb200_error_clear()
    assert rc == -1 and "frame %d:" % k in msg, msg
    assert (out == 0xA5).all()
    dev = torch.full((int(np.prod(shape)),), 0xA5, dtype=torch.uint8, device="cuda")
    assert _sentinel_decode(batch, shape, vb.DEVICE, dev.data_ptr()) == -1
    L.vb200_error_clear()
    torch.cuda.synchronize()
    assert (dev.cpu().numpy() == 0xA5).all()
    assert L.vb200_debug_dz_pool_used() == pool
    assert np.array_equal(vb.png_decode_batch(streams), want)
    assert L.vb200_debug_dz_pool_used() == pool


@pytest.mark.gpu
def test_gpu_chunks(vb):
    """batches split by the device-memory budget decode as one"""
    streams, want = mixed_batch(3, 33, 40)
    L = vb.lib()
    try:
        L.vb200_debug_png_set_budget(3 * 33 * 128)
        assert np.array_equal(vb.png_decode_batch(streams), want)
        L.vb200_debug_png_set_budget(100)
        with pytest.raises(vb.Error, match="more than the 100 allowed"):
            vb.png_decode_batch(streams[:2])
    finally:
        L.vb200_debug_png_set_budget(0)


def _png_of(a, mode=None, **kw):
    b = io.BytesIO()
    PIL.fromarray(a, mode).save(b, "PNG", **kw)
    return b.getvalue()


def thumbnail_cases():
    rng = np.random.default_rng(11)
    h, w = 300, 410
    base = rng.integers(0, 256, (h // 10 + 1, w // 10 + 1, 4), dtype=np.uint8).repeat(10, 0).repeat(10, 1)[:h, :w]
    base[::7] = rng.integers(0, 256, (len(range(0, h, 7)), w, 4), dtype=np.uint8)
    pal = PIL.fromarray(base[:, :, :3]).quantize(64)
    b_pal = io.BytesIO()
    pal.save(b_pal, "PNG")
    b_palt = io.BytesIO()
    pal.save(b_palt, "PNG", transparency=5)
    return {"rgb": _png_of(base[:, :, :3]), "rgba": _png_of(base), "grey": _png_of(base[:, :, 0]), "ga": _png_of(base[:, :, :2], "LA"),
            "pal": b_pal.getvalue(), "pal_trns": b_palt.getvalue()}


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["rgb", "rgba", "grey", "ga", "pal", "pal_trns"])
def test_gpu_thumbnails(vb, oracle, case):
    s = thumbnail_cases()[case]
    dec = vb.png_decode_host_twin(s)
    assert np.array_equal(dec, pillow(s, dec.shape[2]))
    h, w, bands = dec.shape
    for target in (37, 128, 200):
        want = oracle.thumbnail_image(dec, target)
        assert np.array_equal(vb.thumbnail_buffer(s, target), want), (case, target)
        plan = vb.ThumbnailPlan(w, h, bands, target)
        got = plan.run_png([s, s, s])
        plan.close()
        assert np.array_equal(got[2], want), (case, target)


@pytest.mark.gpu
def test_gpu_thumbnail_icc(vb):
    from icc_fixtures import rgb_profile
    prof = bytes(rgb_profile("gamma"))
    a = np.random.default_rng(2).integers(0, 256, (120, 170, 3), dtype=np.uint8)
    s = _png_of(a, icc_profile=prof)
    out_prof = bytes(rgb_profile("srgb"))
    dec = vb.png_decode_host_twin(s)
    want = vb.Image(dec).thumbnail_image(64, output_profile=out_prof, embedded_profile=prof).numpy()
    assert np.array_equal(vb.thumbnail_buffer(s, 64, output_profile=out_prof), want)
    want = vb.Image(dec).thumbnail_image_linear(64, output_profile=out_prof, embedded_profile=prof).numpy()
    assert np.array_equal(vb.thumbnail_buffer_linear(s, 64, output_profile=out_prof), want)
    want = vb.Image(dec).thumbnail_image_linear(64, embedded_profile=prof).numpy()
    assert np.array_equal(vb.thumbnail_buffer_linear(s, 64), want)


@pytest.mark.gpu
def test_gpu_thumbnail_declines_exif(vb):
    a = np.random.default_rng(2).integers(0, 256, (40, 50, 3), dtype=np.uint8)
    exif = PIL.Exif()
    exif[0x0112] = 6
    s = _png_of(a, exif=exif.tobytes())
    assert b"eXIf" in s
    assert np.array_equal(vb.png_decode_batch([s])[0], a)
    with pytest.raises(vb.Error, match="eXIf"):
        vb.thumbnail_buffer(s, 20)
    with pytest.raises(vb.Error, match="eXIf"):
        vb.thumbnail_buffer_linear(s, 20)
    plan = vb.ThumbnailPlan(50, 40, 3, 20)
    with pytest.raises(vb.Error, match="eXIf"):
        plan.run_png([s])
    plan.close()

"""tiff2vips + libtiff restated for the device decoder's subset (test infrastructure).

load(stream, page, n, subifd) is what vips_tiffload_buffer gives for 8-bit, contiguous, FillOrder 1 MINISBLACK /
MINISWHITE / RGB images compressed with none, PackBits, LZW or deflate, with predictor 1 or 2:
  - the IFD walk of rtiff_set_page (tiff2vips.c:798-846): the page's IFD along the chain, then its SubIFD;
  - each strip or tile decoded as libtiff does: zlib for deflate, LZWDecode and PackBitsDecode restated below, a segment
    that decodes short refused ("Not enough data"), then horAcc8 (tif_predict.c) over each row of the segment;
  - rtiff_greyscale_line's inversion of MINISWHITE's first band, everything else copied (rtiff_parse_copy).
pyramid_level restates vips_thumbnail_open's TIFF pyramid search (thumbnail.c:262-383, 519-541, 562-581).
Anything outside the subset raises ValueError.
"""
import zlib

import numpy as np


class Tiff:
    def __init__(self, data):
        self.d = bytes(data)
        if self.d[:2] == b"II":
            self.e = "<"
        elif self.d[:2] == b"MM":
            self.e = ">"
        else:
            raise ValueError("not a TIFF stream")
        magic = self.u(2, 2)
        if magic == 42:
            self.big = False
            off = self.u(4, 4)
        elif magic == 43:
            self.big = True
            off = self.u(8, 8)
        else:
            raise ValueError("not a TIFF stream")
        self.pages = []
        while off:
            self.pages.append(off)
            if len(self.pages) > 65536:
                raise ValueError("IFD loop")
            n = self.u(off, 8 if self.big else 2)
            off = self.u(off + (8 if self.big else 2) + n * (20 if self.big else 12), 8 if self.big else 4)

    def u(self, at, size):
        if at < 0 or at + size > len(self.d):
            raise ValueError("outside the stream")
        return int.from_bytes(self.d[at:at + size], "little" if self.e == "<" else "big")

    def ifd(self, off):
        """{tag: list of ints or bytes}"""
        cb, eb, inl = (8, 20, 8) if self.big else (2, 12, 4)
        sizes = {1: 1, 2: 1, 3: 2, 4: 4, 5: 8, 6: 1, 7: 1, 8: 2, 9: 4, 10: 8, 11: 4, 12: 8, 13: 4, 16: 8, 17: 8, 18: 8}
        tags = {}
        for k in range(self.u(off, cb)):
            e = off + cb + k * eb
            tag, typ = self.u(e, 2), self.u(e + 2, 2)
            count = self.u(e + 4, inl)
            sz = sizes.get(typ, 0)
            if not sz:
                continue
            at = e + 4 + inl
            if count * sz > inl:
                at = self.u(at, inl)
            if at + count * sz > len(self.d):
                raise ValueError("tag %d outside the stream" % tag)
            if typ in (1, 3, 4, 13, 16, 18):
                tags[tag] = [self.u(at + i * sz, sz) for i in range(count)]
            elif typ == 7:
                tags[tag] = self.d[at:at + count]
        return tags

    def select(self, page, subifd):
        if not 0 <= page < len(self.pages):
            raise ValueError("bad page number")
        t = self.ifd(self.pages[page])
        if subifd >= 0:
            subs = t.get(330, [])
            if subifd >= len(subs):
                raise ValueError("subifd out of range")
            t = self.ifd(subs[subifd])
        return t


def lzw_decode(src, want):
    """libtiff's LZWDecode (tif_lzw.c) of one segment into exactly `want` bytes"""
    src = bytes(src)
    nbits, free, bit = 9, 258, 0
    table = {}
    out = bytearray()
    old = None
    total = len(src) * 8

    def code():
        nonlocal bit
        if total - bit < nbits:
            return 257
        v = 0
        for i in range(nbits):
            b = bit + i
            v = (v << 1) | ((src[b >> 3] >> (7 - (b & 7))) & 1)
        bit += nbits
        return v

    def string(c):
        return bytes([c]) if c < 256 else table[c]

    while len(out) < want:
        c = code()
        if c == 257:
            break
        if c == 256:
            while c == 256:
                free, nbits, table = 258, 9, {}
                c = code()
            if c == 257:
                break
            if c > 256:
                raise ValueError("corrupted LZW table")
            out.append(c)
            old = c
            continue
        if old is None or free >= 4095 + 1024 or (c >= 258 and c > free):
            raise ValueError("corrupted LZW table")
        prev = string(old)
        cur_first = string(c)[0] if c != free else prev[0]
        table[free] = prev + bytes([cur_first])
        free += 1
        if free > (1 << nbits) - 2 and nbits < 12:
            nbits += 1
        out += string(c)
        old = c
    if len(out) < want:
        raise ValueError("not enough data")
    return bytes(out[:want])


def packbits_decode(src, want):
    """libtiff's PackBitsDecode (tif_packbits.c)"""
    out = bytearray()
    i = 0
    while i < len(src) and len(out) < want:
        n = src[i]
        i += 1
        if n >= 128:
            n -= 256
        if n < 0:
            if n == -128:
                continue
            n = min(-n + 1, want - len(out))
            if i >= len(src):
                break
            out += bytes([src[i]]) * n
            i += 1
        else:
            n = min(n, want - len(out) - 1)
            if len(src) - i < n + 1:
                break
            out += src[i:i + n + 1]
            i += n + 1
    if len(out) < want:
        raise ValueError("not enough data")
    return bytes(out)


def splice(tables, tile):
    """the stream libjpeg decodes after rtiff_decompress_jpeg_run's tables-only pass (tiff2vips.c:2097-2109): JPEGTables'
    DQT and DHT segments after the tile's SOI"""
    if tables is None:
        return bytes(tile)
    t = bytes(tables)
    if len(t) < 4 or t[:2] != b"\xff\xd8":
        raise ValueError("bad JPEGTables")
    keep, p = b"", 2
    while True:
        if t[p] != 0xFF:
            raise ValueError("bad JPEGTables")
        m = t[p + 1]
        if m == 0xD9:
            break
        n = int.from_bytes(t[p + 2:p + 4], "big")
        if m in (0xDB, 0xC4):
            keep += t[p:p + 2 + n]
        p += 2 + n
    return bytes(tile[:2]) + keep + bytes(tile[2:])


def jpeg_tile(tables, tile, shape):
    """one JPEG tile through Pillow's libjpeg-turbo, as rtiff_decompress_jpeg_run reads it -> uint8 [th, tw, spp]"""
    import io
    from PIL import Image
    im = Image.open(io.BytesIO(splice(tables, tile)))
    if im.mode not in ("L", "RGB"):
        raise ValueError("JPEG tile of mode %s" % im.mode)
    a = np.asarray(im)
    a = a if a.ndim == 3 else a[:, :, None]
    if a.shape != shape:
        raise ValueError("JPEG tile decodes to %s, the tiles are %s" % (a.shape, shape))
    return a


def _segment(comp, data, want):
    if comp == 1:
        if len(data) < want:
            raise ValueError("not enough data")
        return data[:want]
    if comp == 32773:
        return packbits_decode(data, want)
    if comp == 5:
        if len(data) >= 2 and data[0] == 0 and data[1] & 1:
            raise ValueError("old-style LZW")
        return lzw_decode(data, want)
    if comp in (8, 32946):
        z = zlib.decompressobj()
        out = z.decompress(data, want)
        if len(out) < want:
            raise ValueError("not enough data")
        return out
    raise ValueError("compression %d not supported" % comp)


def load_ifd(t, tiff):
    """one IFD's pixels -> uint8 [h, w, spp]"""
    w, h = t[256][0], t[257][0]
    spp = t.get(277, [1])[0]
    bps = t.get(258, [1])
    ph = t.get(262, [None])[0]
    comp = t.get(259, [1])[0]
    pred = t.get(317, [1])[0]
    if any(b != 8 for b in bps) or t.get(339, [1])[0] != 1 or t.get(284, [1])[0] != 1 or t.get(266, [1])[0] != 1:
        raise ValueError("outside the subset")
    if comp == 7 and (322 not in t or ph == 2):
        raise ValueError("JPEG strips / RGB-photometric JPEG")
    if not ((ph in (0, 1) and spp in (1, 2)) or (ph == 2 and spp in (3, 4)) or (ph == 6 and comp == 7 and spp == 3)):
        raise ValueError("photometric %s with %d samples" % (ph, spp))
    if t.get(338, [0])[0] not in (0, 2) or pred not in (1, 2):
        raise ValueError("extra samples / predictor")
    use_pred = pred == 2 and comp in (5, 8, 32946)
    if 322 in t:
        tw, th = t[322][0], t[323][0]
        offs, counts = t[324], t[325]
        across = (w + tw - 1) // tw
        segs = [(k, (k % across) * tw, (k // across) * th, tw, th) for k in range(across * ((h + th - 1) // th))]
    else:
        rps = max(1, min(t.get(278, [2 ** 32 - 1])[0], h))
        offs, counts = t[273], t[279]
        segs = [(k, 0, k * rps, w, min(rps, h - k * rps)) for k in range((h + rps - 1) // rps)]
    out = np.zeros((h, w, spp), np.uint8)
    for k, x0, y0, sw, sh in segs:
        o, c = offs[k], counts[k]
        if o + c > len(tiff.d):
            raise ValueError("segment outside the stream")
        if comp == 7:
            a = jpeg_tile(t.get(347), tiff.d[o:o + c], (sh, sw, spp))
        else:
            raw = _segment(comp, tiff.d[o:o + c], sw * sh * spp)
            a = np.frombuffer(raw, np.uint8).reshape(sh, sw, spp)
        if use_pred:
            a = np.cumsum(a.astype(np.uint64), axis=1).astype(np.uint8)
        cw, ch = min(sw, w - x0), min(sh, h - y0)
        out[y0:y0 + ch, x0:x0 + cw] = a[:ch, :cw]
    if ph == 0:  # WhiteIsZero
        out[..., 0] = 255 - out[..., 0]
    return out


def load(stream, page=0, n=1, subifd=-1):
    """vips_tiffload_buffer(page=page, n=n, subifd=subifd) -> uint8 [h * n, w, bands]"""
    tiff = Tiff(stream)
    if n == -1:
        n = len(tiff.pages) - page
    return np.concatenate([load_ifd(tiff.select(p, subifd), tiff) for p in range(page, page + n)], axis=0)


def icc_profile(stream, page=0, subifd=-1):
    t = Tiff(stream).select(page, subifd)
    return t.get(34675)


def pyramid_level(input_w, input_h, pages, subifds, width, height, size="both"):
    """(subifd, page) of vips_thumbnail_open's TIFF branch: pages / subifds are the (w, h) of every page's main IFD and of
    page 0's SubIFDs; (-1, 0) without a pyramid"""
    def detect(levels, sub):
        for i, (lw, lh) in enumerate(levels):
            ew = input_w // (2 << i) if sub else input_w // (1 << i)
            eh = input_h // (2 << i) if sub else input_h // (1 << i)
            if abs(lw - ew) > 5 or lw < 2 or abs(lh - eh) > 5 or lh < 2:
                return None
        return levels

    found, sub = None, True
    if 1 <= len(subifds) <= 28:
        found = detect(subifds, True)
    if found is None:
        sub = False
        if 2 <= len(pages) <= 29:
            found = detect(pages, False)
    if found is None:
        return -1, 0
    level = 0
    for l in range(len(found) - 1, -1, -1):
        if common_shrink(found[l][0], found[l][1], width, height, size) > 1.0:
            level = l
            break
    return (level, 0) if sub else (-1, level)


def common_shrink(w, h, tw, th, size="both"):
    """vips_thumbnail_calculate_common_shrink (thumbnail.c:469-485) over vips_thumbnail_calculate_shrink (:413-466), no
    crop and no rotation"""
    th = th or tw
    hs, vs = w / tw, h / th
    if size != "force":
        if hs < vs:
            hs = vs
        else:
            vs = hs
    if size == "up":
        hs, vs = min(1, hs), min(1, vs)
    elif size == "down":
        hs, vs = max(1, hs), max(1, vs)
    return min(min(hs, w), min(vs, h))


def level_geometry(stream):
    """(input w, h, [page (w, h)], [subifd (w, h)]) as vips_thumbnail_open reads them"""
    tiff = Tiff(stream)
    t0 = tiff.ifd(tiff.pages[0])
    pages = []
    for p in tiff.pages:
        t = tiff.ifd(p)
        pages.append((t[256][0], t[257][0]))
    subs = []
    for o in t0.get(330, []):
        t = tiff.ifd(o)
        subs.append((t[256][0], t[257][0]))
    return t0[256][0], t0[257][0], pages, subs


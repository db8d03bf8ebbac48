"""tools/fuzz_host_parsers.py -- mutation fuzzing of the host-side parsers that read untrusted bytes (the JPEG marker
parser + the decoder's host twin, the embedded-ICC-profile reader, the ICC profile parser, the GIF block walker + the GIF
decoder's host twin with its LZW, the PNG chunk walker + the PNG
decoder's host twin with its inflate, on PNG streams and on raw deflate data, the TIFF IFD walk + the TIFF decoder's host
twin with its LZW and PackBits and the pyramid-level search, the WebP RIFF / VP8X / frame-tag parser + the VP8 decoder's
host twin), meant to run against an AddressSanitizer build:

    VB200_LIB=/tmp/asan/libvb200_asan.so LD_PRELOAD=$(gcc -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 \
        python tools/fuzz_host_parsers.py [seconds]

Every call must either succeed or fail with vb.Error; a crash or an ASan report is a bug.  No GPU is used."""
import io
import sys
import time
import zlib

import numpy as np
from PIL import Image as PIL

sys.path.insert(0, __file__.rsplit("/tools/", 1)[0])
sys.path.insert(0, __file__.rsplit("/tools/", 1)[0] + "/tests")
import libvips_b200 as vb  # noqa: E402


def jpegs(rng):
    out = []
    for shape in ((33, 47, 3), (64, 64, 3), (17, 90, 1)):
        a = rng.integers(0, 256, shape, dtype=np.uint8)
        if shape[2] == 1:
            a = a[:, :, 0]
        for kw in (dict(), dict(subsampling=0), dict(subsampling=1), dict(progressive=True), dict(restart_marker_blocks=2),
                   dict(progressive=True, restart_marker_blocks=3), dict(optimize=True)):
            if a.ndim == 2:
                kw = {k: v for k, v in kw.items() if k != "subsampling"}
            b = io.BytesIO()
            PIL.fromarray(a).save(b, "JPEG", quality=int(rng.integers(30, 96)), **kw)
            out.append(b.getvalue())
    return out


def pngs(rng):
    out = []
    for mode, shape, kw in (("RGB", (33, 47, 3), {}), ("RGBA", (20, 9, 4), {}), ("L", (17, 90), {}), ("LA", (5, 31, 2), {}),
                            ("P", (29, 13), {"bits": 2}), ("P", (40, 40), {"transparency": 1}), ("L", (8, 8), {"transparency": 3}),
                            ("RGB", (9, 9, 3), {"icc_profile": bytes(range(256)) * 2})):
        a = rng.integers(0, 4 if mode == "P" else 256, shape, dtype=np.uint8)
        a[: shape[0] // 2] = a[:1]
        b = io.BytesIO()
        PIL.fromarray(a, mode).save(b, "PNG", compress_level=int(rng.integers(0, 10)), **kw)
        out.append(b.getvalue())
    return out


def mutate(rng, s):
    s = bytearray(s)
    k = rng.integers(0, 6)
    if k == 0:
        return bytes(s[: rng.integers(0, len(s))])
    if k == 1:
        for _ in range(rng.integers(1, 8)):
            s[rng.integers(0, len(s))] ^= 1 << rng.integers(0, 8)
    elif k == 2:  # damage a marker segment length
        pos = [i for i in range(len(s) - 3) if s[i] == 0xFF and 0xC0 <= s[i + 1] <= 0xFE]
        if pos:
            i = pos[rng.integers(0, len(pos))]
            s[i + 2] = rng.integers(0, 256)
            s[i + 3] = rng.integers(0, 256)
    elif k == 3:
        i = rng.integers(0, len(s))
        s[i:i] = bytes(rng.integers(0, 256, rng.integers(1, 40), dtype=np.uint8))
    elif k == 4:
        i = rng.integers(0, len(s))
        del s[i:i + rng.integers(1, 60)]
    else:
        i = rng.integers(0, len(s))
        n = rng.integers(1, 30)
        s[i:i + n] = bytes(rng.integers(0, 256, n, dtype=np.uint8))
    return bytes(s)


def app2_mutant(rng, s):
    """a JPEG with APP2 ICC_PROFILE segments in any order: sequence numbers 0 / 1 / 100 / 101 / 255 and random, duplicates,
    gaps, segment lengths 13 .. 16, and segments after the first SOS"""
    segs = []
    for _ in range(rng.integers(0, 6)):
        seq = int(rng.choice([0, 1, 2, 3, 100, 101, 255, rng.integers(0, 256)]))
        body = b"ICC_PROFILE\0" + bytes([seq, int(rng.integers(0, 256))]) + bytes(rng.integers(0, 256, rng.integers(0, 300), dtype=np.uint8))
        body = body[:int(rng.choice([13, 14, 15, 16, len(body)]))]
        segs.append(b"\xff\xe2" + (len(body) + 2).to_bytes(2, "big") + body)
    cut = 2 if rng.integers(0, 2) else max(2, s.find(b"\xff\xda") + 4 + int(rng.integers(0, 40)))
    return s[:cut] + b"".join(segs) + s[cut:]


def gifs(rng):
    """GIFs written by Pillow: static and animated, with and without transparency, interlaced or not"""
    out = []
    for i in range(6):
        h, w = int(rng.integers(1, 60)), int(rng.integers(1, 60))
        ims = [PIL.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8)).quantize(int(rng.integers(2, 257))) for _ in range(1 + i % 3)]
        b = io.BytesIO()
        kw = {"transparency": 1} if i % 2 else {}
        ims[0].save(b, "GIF", save_all=True, append_images=ims[1:], interlace=bool(i % 4 == 3), disposal=i % 4, **kw)
        out.append(b.getvalue())
    return out


def tiffs(rng):
    """TIFFs from the test-suite's writer (BigTIFF, both byte orders, tiles, pages, SubIFDs) and from Pillow's libtiff"""
    import test_tiff as TT
    out = []
    for i in range(8):
        a = rng.integers(0, 256, (int(rng.integers(1, 40)), int(rng.integers(1, 40)), (1, 2, 3, 4)[i % 4]), dtype=np.uint8)
        comp = (1, 32773, 5, 8)[i % 4]
        kw = dict(tile=(16, 16)) if i % 2 else dict(rps=int(rng.integers(1, 9)))
        out.append(TT.make_tiff([TT.Page(a, comp=comp, pred=1 + (i % 3 == 0), subifds=[TT.Page(a[::2, ::2], comp=comp)], icc=b"icc" * 9,
                                         **kw)] * (1 + i % 3), "<>"[i % 2], i % 3 == 1))
    for comp in ("tiff_lzw", "packbits", "tiff_adobe_deflate"):
        b = io.BytesIO()
        PIL.fromarray(rng.integers(0, 256, (23, 31, 3), dtype=np.uint8)).save(b, "TIFF", compression=comp)
        out.append(b.getvalue())
    return out


def webps(rng):
    """lossy WebPs from Pillow's libwebp (simple format, and VP8X with an ICCP chunk) and the test-suite's VP8 key-frame
    writer (2 / 4 / 8 partitions, segments, filter deltas)"""
    import test_webp as TW
    out = []
    for i in range(6):
        a = rng.integers(0, 256, (int(rng.integers(1, 40)), int(rng.integers(1, 40)), 3), dtype=np.uint8)
        b = io.BytesIO()
        PIL.fromarray(a).save(b, "WEBP", quality=int(rng.integers(0, 101)), **({"icc_profile": b"icc" * 9} if i % 2 else {}))
        out.append(b.getvalue())
    out += [TW.vp8_stream(int(rng.integers(0, 1 << 30)), h=int(rng.integers(1, 40)), w=int(rng.integers(1, 40))) for _ in range(6)]
    return out


def main():
    budget = float(sys.argv[1]) if len(sys.argv) > 1 else 60.0
    rng = np.random.default_rng(int(time.time()))
    good = jpegs(rng)
    good_png = pngs(rng)
    good_gif = gifs(rng)
    good_tiff = tiffs(rng)
    good_webp = webps(rng)
    lzw = [g[g.index(b"\x2c") + 11:] for g in good_gif]  # from the minimum code size on: sub-block framing fed to the LZW as data
    deflate = [zlib.compress(s, int(rng.integers(0, 10)))[2:-4] for s in good_png]
    import icc_fixtures as F
    import test_icc as T
    profiles = [F.rgb_profile(t) for t in ("srgb", "gamma", "para4", "table")] + [F.grey_profile(), F.ink_profile(),
                                                                               F.lut_v4_rgb_profile("XYZ "), F.lut_v4_rgb_profile("Lab ")]
    profiles = [bytes(p) for p in profiles]
    t0 = time.time()
    n = fails = ok = 0
    px = rng.integers(0, 256, (16, 3), dtype=np.uint8)
    while time.time() - t0 < budget:
        s = mutate(rng, good[rng.integers(0, len(good))])
        for shrink in (1, 2, 8):
            try:
                vb.jpeg_decode_host_twin(s, shrink)
                ok += 1
            except vb.Error:
                fails += 1
        for t in (s, app2_mutant(rng, good[rng.integers(0, len(good))])):
            try:
                vb.jpeg_icc_profile(t)
                ok += 1
            except vb.Error:
                fails += 1
        p = mutate(rng, good_png[rng.integers(0, len(good_png))])
        for fn in (vb.png_decode_host_twin, vb.png_icc_profile, lambda t: vb.png_geometry([t])):
            try:
                fn(p)
                ok += 1
            except vb.Error:
                fails += 1
        g = mutate(rng, good_gif[rng.integers(0, len(good_gif))])
        for fn in (vb.gif_decode_host_twin, lambda t: vb.gif_decode_host_twin(t, 0, -1), vb.gif_geometry):
            try:
                fn(g)
                ok += 1
            except vb.Error:
                fails += 1
        t = mutate(rng, good_tiff[rng.integers(0, len(good_tiff))])
        for fn in (vb.tiff_decode_host_twin, lambda t: vb.tiff_decode_host_twin(t, 0, -1, 0), lambda t: vb.tiff_geometry(t, 0, 0),
                   vb.tiff_icc_profile, lambda t: vb.thumbnail_tiff_level(t, 5), lambda t: vb.tiff_lzw_host_twin(t[8:], 1 << 12)):
            try:
                fn(t)
                ok += 1
            except vb.Error:
                fails += 1
        w = mutate(rng, good_webp[rng.integers(0, len(good_webp))])
        for fn in (vb.webp_decode_host_twin, vb.webp_geometry, vb.webp_icc_profile):
            try:
                fn(w)
                ok += 1
            except vb.Error:
                fails += 1
        try:
            vb.lzw_host_twin(mutate(rng, lzw[rng.integers(0, len(lzw))]), int(rng.integers(0, 13)), 1 << 14, bool(rng.integers(0, 2)))
            ok += 1
        except vb.Error:
            fails += 1
        try:
            vb.inflate_host_twin(mutate(rng, deflate[rng.integers(0, len(deflate))]), 1 << 16)
            ok += 1
        except vb.Error:
            fails += 1
        if profiles:
            p = mutate(rng, profiles[rng.integers(0, len(profiles))])
            for mode in (0, 1):
                try:
                    T.host_eval(mode, px if mode == 0 else px.astype(np.float32), p, intent=int(rng.integers(0, 4)), pcs=int(rng.integers(0, 2)))
                    ok += 1
                except vb.Error:
                    fails += 1
        n += 1
    print("fuzz: %d mutants, %d calls ok, %d rejected, %d profiles, no crash" % (n, ok, fails, len(profiles)))


if __name__ == "__main__":
    main()

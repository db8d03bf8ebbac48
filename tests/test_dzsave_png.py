"""Deep Zoom / Zoomify pyramids with PNG tiles (vb200_dzsave_png, csrc/dzsave.cu) against vips_dzsave with suffix ".png".

The reference writes each tile with vips_image_write_to_buffer(tile, ".png") (dzsave.c write_image :369-402): spngsave with
its defaults and keep NONE.  An image with alpha (vips_image_hasalpha: 2-band B_W, 4-band sRGB) is shrunk by
vips_region_shrink_alpha (iofuncs/region.c:1444-1482), which works in double; the library states it in integers.  Three
statements of that shrink are held against each other here: the reference's own macro (extracted from region.c and compiled
into oracle/_ref/libregion_shrink.so where the reference is present), oracle/pydz_alpha.py's restatement in double, and the
library's per-pixel code (the host twin).  oracle/pydz_alpha.py's strip walk (oracle/pydz.py's, with the alpha shrink) is
held against the library's whole-image
pyramid, and every tile's IDAT payload against Python's zlib over scanlines built from the PNG specification
(tests/test_png_save_options.py).

CPU tests run the kernels' per-pixel code and the encoder's host twin (vb200_debug_dzsave_png); -m gpu tests the kernels.
"""
import ctypes as C
import io
import os
import threading

import numpy as np
import pytest

PIL = pytest.importorskip("PIL.Image")

from test_dzsave import GRID, noise, pyramid_levels, same_pyramid  # noqa: E402
from test_png_save_options import chunks, idat, low_bit_expected, scan_rows, zlib_stream  # noqa: E402

from oracle import pydz_alpha  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REGION_SHRINK = os.path.join(ROOT, "oracle", "_ref", "libregion_shrink.so")
ZLIB_STRATEGY = {"default": 0, "filtered": 1}
ALPHAS = [0, 1, 2, 3, 4, 127, 128, 129, 253, 254, 255]


@pytest.fixture(scope="module")
def vb():
    import libvips_b200 as vb
    vb.lib()
    return vb


def alpha_pyramid_levels(a):
    """the whole-image statement with alpha in numpy, from the top: the integer form of vips_region_shrink_alpha"""
    out = [a]
    while out[-1].shape[0] > 1 or out[-1].shape[1] > 1:
        p = out[-1].astype(np.int64)
        if p.shape[0] & 1:
            p = np.concatenate([p, p[-1:]], 0)
        if p.shape[1] & 1:
            p = np.concatenate([p, p[:, -1:]], 1)
        q = [p[0::2, 0::2], p[0::2, 1::2], p[1::2, 0::2], p[1::2, 1::2]]
        S = sum(x[..., -1:] for x in q)
        num = sum(x[..., :-1] * x[..., -1:] for x in q)
        level = np.concatenate([num // np.maximum(S, 1), S >> 2], -1)
        out.append(np.where(S == 0, 0, level).astype(np.uint8))
    return out


def levels_of(a):
    return alpha_pyramid_levels(a) if a.shape[2] in (2, 4) else pyramid_levels(a)


def quads_image(q):
    """quads [n, 4, bands] (p00, p01, p10, p11) -> a 2 x 2n image whose level 1 is one pixel per quad"""
    n, _, bands = q.shape
    return q.reshape(n, 2, 2, bands).transpose(1, 0, 2, 3).reshape(2, 2 * n, bands)


def region_shrink_oracle():
    if not os.path.exists(REGION_SHRINK):
        pytest.skip("oracle/_ref/libregion_shrink.so not built (needs the reference's region.c)")
    L = C.CDLL(REGION_SHRINK)
    for fn in (L.region_shrink_alpha_uchar, L.region_shrink_mean_uchar):
        fn.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
        fn.restype = None
    return L


def reference_shrink(L, img, alpha=True):
    """the reference's macro over a 2 x 2n image -> 1 x n"""
    img = np.ascontiguousarray(img)
    _, w2, bands = img.shape
    out = np.empty((1, w2 // 2, bands), np.uint8)
    fn = L.region_shrink_alpha_uchar if alpha else L.region_shrink_mean_uchar
    fn(img.ctypes.data, w2 * bands, w2 // 2, bands, out.ctypes.data)
    return out


def alpha_quads(bands, seed):
    """every alpha quad over ALPHAS^4 with random colours, then 10^6 random quads"""
    rng = np.random.default_rng(seed)
    grid = np.array(np.meshgrid(*[ALPHAS] * 4, indexing="ij")).reshape(4, -1).T
    q = rng.integers(0, 256, (len(grid), 4, bands), dtype=np.uint8)
    q[..., -1] = grid
    return np.concatenate([q, rng.integers(0, 256, (10 ** 6, 4, bands), dtype=np.uint8)])


# ---------------------------------------------------------------------------------------------------------------- CPU

@pytest.mark.parametrize("bands", [2, 4])
def test_alpha_shrink_restatement_equals_the_library(vb, bands):
    q = alpha_quads(bands, bands)
    img = quads_image(q)
    want = pydz_alpha.shrink_alpha(img[0:1, 0::2], img[0:1, 1::2], img[1:2, 0::2], img[1:2, 1::2])
    got = vb.dz_pyramid_level_host_twin(img, 1)
    assert np.array_equal(got, want)
    assert np.array_equal(got, alpha_pyramid_levels(img)[1])
    # S = 0: every band 0, whatever the colours
    zero = got[0, :len(ALPHAS) ** 4][(q[:len(ALPHAS) ** 4, :, -1].astype(int).sum(1) == 0)]
    assert len(zero) == 1 and not zero.any()
    # one non-zero alpha: the colour is that pixel's own, the alpha a quarter of it
    one = np.zeros((4, 4, bands), np.uint8)
    one[..., :-1] = np.arange(16 * (bands - 1)).reshape(4, 4, bands - 1) * 7 % 256
    for k in range(4):
        one[k, k, -1] = (1, 3, 128, 255)[k]
        assert np.array_equal(vb.dz_pyramid_level_host_twin(quads_image(one[k:k + 1]), 1)[0, 0],
                              np.append(one[k, k, :-1], (1, 3, 128, 255)[k] >> 2))


def test_alpha_shrink_is_the_reference_macro(vb):
    L = region_shrink_oracle()
    for bands in (2, 4):
        img = quads_image(alpha_quads(bands, 10 + bands))
        ref = reference_shrink(L, img)
        assert np.array_equal(ref, pydz_alpha.shrink_alpha(img[0:1, 0::2], img[0:1, 1::2], img[1:2, 0::2], img[1:2, 1::2])), bands
        assert np.array_equal(ref, vb.dz_pyramid_level_host_twin(img, 1)), bands
    # the mean macro is the JPEG path's shrink
    img = quads_image(np.random.default_rng(3).integers(0, 256, (20000, 4, 3), dtype=np.uint8))
    assert np.array_equal(reference_shrink(L, img, alpha=False), vb.dz_pyramid_level_host_twin(img, 1))


def test_opaque_rgba_is_not_the_rgb_pyramid(vb):
    """alpha 255 everywhere: floor(sum / 4) per colour band, where the mean path rounds (sum + 2) >> 2"""
    a = noise(64, 64, 4, 1)
    a[..., 3] = 255
    got = vb.dz_pyramid_level_host_twin(a, 1)
    rgb = vb.dz_pyramid_level_host_twin(np.ascontiguousarray(a[..., :3]), 1)
    p = a[..., :3].astype(np.int32)
    s = p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2]
    assert np.array_equal(got[..., :3], s // 4) and np.array_equal(rgb, (s + 2) >> 2)
    assert (got[..., :3] != rgb).any() and (got[..., 3] == 255).all()


def alpha_grid():
    """test_dzsave's grid with 2 and 4 bands in place of 1 and 3, every third case"""
    return [(c[0], c[1], c[2] + 1) + tuple(c[3:]) for c in GRID[::3]]


@pytest.mark.parametrize("case", alpha_grid(), ids=lambda c: "%dx%dx%d-%d_%d-%s-%s" % (c[0], c[1], c[2], c[3][0], c[3][1], c[4], c[5]))
def test_strip_walk_with_alpha_is_the_whole_image_statement(vb, case):
    w, h, bands, (tile_size, overlap), depth, layout = case
    a = noise(h, w, bands, w * 29 + h)
    a[..., -1] = np.where(a[..., -1] < 64, 0, a[..., -1])           # transparent pixels, so S = 0 occurs
    walk = pydz_alpha.dzsave(a, layout, tile_size, overlap, depth, "im", suffix=".png")
    got = vb.dzsave_png_host_twin(a, "im", layout=layout, tile_size=tile_size, overlap=overlap, depth=depth, compression=4)
    assert [(n,) + g for n, g in enumerate(got.levels)] == walk.levels()
    want = sorted(walk.tiles, key=lambda t: (t[1], t[3], t[2]))
    assert len(got.tiles) == len(want)
    levels = levels_of(a)
    top = len(got.levels) - 1
    for t, (name, n, x, y, rect, pixels) in zip(got.tiles, want):
        assert (t.name, t.level, t.x, t.y, t.rect) == (name, n, x, y, rect)
        left, tp, tw, th = rect
        assert np.array_equal(levels[top - n][tp:tp + th, left:left + tw], pixels), name
    assert got.sidecar == walk.sidecar()
    # the tiles of the smallest levels decode to the walk's pixels
    for t, (name, n, x, y, rect, pixels) in list(zip(got.tiles, want))[:6]:
        assert np.array_equal(np.asarray(PIL.open(io.BytesIO(t.bytes))).reshape(pixels.shape), pixels), name


COLOUR_TYPE = {1: 0, 2: 4, 3: 2, 4: 6}
OPTIONS = ([dict(bands=b) for b in (1, 2, 3, 4)] + [dict(bands=4, compression=c) for c in (4, 9)] + [dict(bands=3, strategy="filtered")] +
           [dict(bands=2, filter=f) for f in ("sub", "up", "avg", "paeth")] + [dict(bands=4, interlace=True, filter="paeth")] +
           [dict(bands=1, bitdepth=d) for d in (1, 2, 4)] + [dict(bands=3, xres=2.835)])


def check_tiles(p, a, kw):
    """every tile: its chunks, IHDR, pHYs, its IDAT payload as Python's zlib writes it, and Pillow's decode"""
    level, strategy, filt = kw.get("compression", 6), kw.get("strategy", "default"), kw.get("filter", "none")
    interlace, depth, bands = kw.get("interlace", False), kw.get("bitdepth", 8), a.shape[2]
    levels = levels_of(a)
    top = len(p.levels) - 1
    for t in p.tiles:
        left, tp, w, h = t.rect
        pix = levels[top - t.level][tp:tp + h, left:left + w]
        ch = chunks(t.bytes)
        kinds = [k for k, _ in ch]
        assert kinds[0] == b"IHDR" and kinds[1] == b"pHYs" and kinds[-1] == b"IEND" and b"iCCP" not in kinds, t.name
        ihdr = ch[0][1]
        assert ihdr == (w.to_bytes(4, "big") + h.to_bytes(4, "big") + bytes([depth, COLOUR_TYPE[bands], 0, 0, int(interlace)])), t.name
        ppm = int(np.rint(kw.get("xres", 1.0) * 1000)).to_bytes(4, "big")
        assert ch[1][1] == ppm + ppm + b"\x01", t.name
        assert idat(t.bytes) == zlib_stream(b"".join(scan_rows(pix, filt, interlace, depth)), level, ZLIB_STRATEGY[strategy]), t.name
        got = np.asarray(PIL.open(io.BytesIO(t.bytes)).convert({1: "L", 2: "LA", 3: "RGB", 4: "RGBA"}[bands]))
        want = pix if depth == 8 else low_bit_expected(pix, depth)[..., None]
        assert np.array_equal(got.reshape(want.shape), want), t.name


@pytest.mark.parametrize("kw", OPTIONS, ids=lambda o: "-".join("%s=%s" % kv for kv in sorted(o.items())))
def test_host_twin_tiles_are_zlibs_streams(vb, kw):
    kw = dict(kw)
    bands = kw.pop("bands")
    a = noise(150, 230, bands, bands)
    a[40:80, 50:120, -1] = 0
    for layout, tile in (("dz", 64), ("zoomify", 100)):
        check_tiles(vb.dzsave_png_host_twin(a, "t", layout=layout, tile_size=tile, **kw), a, kw)


def test_names_sidecar_and_tree(vb, tmp_path):
    a = noise(300, 520, 4, 4)
    p = vb.dzsave_png_host_twin(a, "slide")
    assert p.tiles[-1].name == "slide_files/10/2_1.png"
    assert 'Format="png"' in p.sidecar[1] and p.sidecar[0] == "slide.dzi"
    assert vb.dzsave_png_host_twin(a, suffix=".PNG").tiles[0].name == "untitled_files/0/0_0.PNG"
    z = vb.dzsave_png_host_twin(a, "z", layout="zoomify")
    assert [t.name for t in z.tiles[:2]] == ["z/TileGroup0/0-0-0.png", "z/TileGroup0/1-0-0.png"]
    p.write(str(tmp_path))
    assert sorted(os.listdir(tmp_path / "slide_files" / "10")) == ["0_0.png", "0_1.png", "1_0.png", "1_1.png", "2_0.png", "2_1.png"]
    im = PIL.open(tmp_path / "slide_files" / "10" / "2_1.png")
    assert im.mode == "RGBA" and im.size == (520 - 507, 300 - 253)
    assert np.array_equal(np.asarray(im), a[253:, 507:])
    assert PIL.open(tmp_path / "slide_files" / "0" / "0_0.png").size == (1, 1)
    z.write(str(tmp_path / "z"))
    assert sorted(os.listdir(tmp_path / "z" / "z")) == ["ImageProperties.xml", "TileGroup0"]
    assert PIL.open(tmp_path / "z" / "z" / "TileGroup0" / "0-0-0.png").mode == "RGBA"


def test_declines(vb):
    L = vb.lib()
    a = noise(40, 30, 4, 0)
    refused = [({"suffix": ".jpeg"}, r"suffix \.jpeg not supported on the device path"),
               ({"suffix": ".webp"}, r"suffix \.webp not supported on the device path"),
               ({"suffix": ".png[compression=9]"}, "suffix options not supported on the device path"),
               ({"compression": 3}, "compression 3 is not built"),
               ({"region_shrink": "median"}, "region_shrink other than mean not supported on the device path"),
               ({"layout": "google"}, "layout google not supported"),
               ({"skip_blanks": 5}, "skip_blanks not supported"),
               ({"container": "zip"}, "zip containers not supported")]
    cases = [(a, kw, m) for kw, m in refused]
    cases += [(noise(8, 8, 3, 0), {"bitdepth": 4}, "bitdepth 4 with 3 bands"),
              (noise(8, 8, 5, 0), {}, "5-band images not supported on the device path"),
              (noise(8, 8, 4, 0).astype(np.uint16), {}, "band format 2 not supported on the device path")]
    before, pool = vb.launch_count(), L.vb200_debug_dz_pool_used()
    for img, kw, message in cases:
        for fn in (vb.dzsave_png, vb.dzsave_png_host_twin):
            with pytest.raises(vb.Error, match=message):
                fn(img, **kw)
    # a Type that is not B_W for 1-2 bands or sRGB for 3-4: spngsave would convert the colours
    for bands, bad in ((4, 1), (3, 0), (2, 22), (1, 22)):
        cin, keep = vb._dz_image(noise(8, 8, bands, 0), None, None, None)
        cin.Type = bad
        handle = C.c_void_p(1)
        for fn in (L.vb200_dzsave_png, L.vb200_debug_dzsave_png):
            assert fn(C.byref(cin), None, None, C.byref(handle)) == -1 and handle.value is None
            assert b"not supported on the device path (PNG tiles take B_W with 1-2 bands, sRGB with 3-4)" in L.vb200_error_buffer()
            L.vb200_error_clear()
    assert vb.launch_count() == before and L.vb200_debug_dz_pool_used() == pool
    # vb200_dzsave keeps its declines
    with pytest.raises(vb.Error, match=r"suffix \.png not supported on the device path"):
        vb.dzsave_host_twin(noise(8, 8, 3, 0), suffix=".png")
    with pytest.raises(vb.Error, match="4-band images not supported on the device path"):
        vb.dzsave_host_twin(a)
    # options NULL and png NULL are the defaults
    cin, keep = vb._dz_image(a, None, None, None)
    handle = C.c_void_p()
    assert L.vb200_debug_dzsave_png(C.byref(cin), None, None, C.byref(handle)) == 0
    got = vb.DzPyramid(handle, None)
    assert [t.bytes for t in got.tiles] == [t.bytes for t in vb.dzsave_png_host_twin(a).tiles]


def test_abi(vb):
    assert C.sizeof(vb.DzOptions) == 64 and C.sizeof(vb.PngSaveOptions) == 32
    L = C.CDLL(vb.library_path())
    for name in ("vb200_dzsave_png", "vb200_debug_dzsave_png", "vb200_dzsave", "vb200_debug_dzsave"):
        assert hasattr(L, name), name


def test_pyramid_level_takes_alpha(vb):
    for (h, w, bands) in ((7, 9, 4), (1, 6, 2), (6, 1, 4), (64, 65, 2), (129, 127, 4)):
        a = noise(h, w, bands, h * w)
        for n, want in enumerate(alpha_pyramid_levels(a)):
            assert np.array_equal(vb.dz_pyramid_level_host_twin(a, n), want), (h, w, bands, n)


# ------------------------------------------------------------------ GPU

def rgba_photo(h, w, seed):
    """smooth colours, a soft alpha edge and a transparent hole"""
    yy, xx = np.mgrid[0:h, 0:w]
    rng = np.random.default_rng(seed)
    rgb = np.stack([128 + 100 * np.sin(xx / 37 + yy / 91), 128 + 90 * np.cos(xx / 53 - yy / 29), (xx * 3 + yy * 5) % 256], -1)
    alpha = np.clip((xx + yy) * 255.0 / max(1, w + h - 2) * 2 - 60, 0, 255)
    a = np.concatenate([rgb, alpha[..., None]], -1) + rng.normal(0, 3, (h, w, 4))
    a = np.clip(a, 0, 255).astype(np.uint8)
    a[h // 3:h // 2, w // 3:w // 2, 3] = 0
    return a


@pytest.mark.gpu
def test_gpu_equals_the_host_twin(vb):
    import torch
    vb.init(0)
    opts = [{}, {"compression": 9, "strategy": "filtered"}, {"filter": "paeth"}, {"interlace": True}, {"filter": "sub", "compression": 4},
            {"filter": "up"}, {"filter": "avg", "xres": 3.0}]
    for k, (w, h, _, (tile_size, overlap), depth, layout) in enumerate(GRID[::4]):
        bands = 1 + k % 4
        a = noise(h, w, bands, w + h)
        kw = dict(layout=layout, tile_size=tile_size, overlap=overlap, depth=depth, **opts[k % len(opts)])
        want = vb.dzsave_png_host_twin(a, "g", **kw)
        same_pyramid(vb.dzsave_png(a, "g", **kw), want, ("host", w, h, bands, kw))
        d = torch.from_numpy(a).cuda()
        same_pyramid(vb.dzsave_png(None, "g", in_ptr=d.data_ptr(), shape=a.shape, **kw), want, ("device", w, h, bands, kw))
    a = noise(40, 70, 1, 1)
    for d in (1, 2, 4):
        same_pyramid(vb.dzsave_png(a, bitdepth=d), vb.dzsave_png_host_twin(a, bitdepth=d), ("bitdepth", d))
    for (w, h) in ((4096, 4096), (5000, 3000)):
        a = rgba_photo(h, w, w)
        want = vb.dzsave_png_host_twin(a, "big")
        same_pyramid(vb.dzsave_png(a, "big"), want, ("host", w, h))
        d = torch.from_numpy(a).cuda()
        same_pyramid(vb.dzsave_png(None, "big", in_ptr=d.data_ptr(), shape=a.shape), want, ("device", w, h))
        for t in want.tiles[-40:]:
            left, tp, tw, th = t.rect
            assert np.array_equal(np.asarray(PIL.open(io.BytesIO(t.bytes))), a[tp:tp + th, left:left + tw]), t.name
    a = noise(300, 400, 4, 5)
    same_pyramid(vb.Image(a).dzsave_png("im", layout="zoomify"), vb.dzsave_png_host_twin(a, "im", layout="zoomify"), "Image.dzsave_png")


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(4097, 4095, 4), (1000, 999, 2), (65537, 3, 4), (3, 65537, 2), (65537, 3, 2), (3, 65537, 4)],
                         ids=lambda s: "%dx%dx%d" % s)
def test_gpu_pyramid_levels_with_alpha(vb, size):
    import torch
    vb.init(0)
    w, h, bands = size
    a = noise(h, w, bands, w + h)
    a[..., -1] = np.where(a[..., -1] < 50, 0, a[..., -1])
    d = torch.from_numpy(a).cuda()
    for n, want in enumerate(alpha_pyramid_levels(a)):
        assert np.array_equal(vb.dz_pyramid_level(None, n, in_ptr=d.data_ptr(), shape=a.shape), want), (size, n)
        if n % 3 == 1:
            assert np.array_equal(vb.dz_pyramid_level(a, n), want), (size, n, "host")


@pytest.mark.gpu
def test_gpu_strides_budget_threads_and_pool(vb):
    import torch
    vb.init(0)
    L = vb.lib()
    a = rgba_photo(600, 700, 6)
    want = vb.dzsave_png_host_twin(a)
    # rows 2807 bytes apart, the first pixel 5 bytes into the allocation: no 16-byte load is legal
    buf = torch.zeros(5 + 600 * 2807, dtype=torch.uint8, device="cuda")
    buf[5:].view(600, 2807)[:, :2800] = torch.from_numpy(a.reshape(600, 2800)).cuda()
    same_pyramid(vb.dzsave_png(None, in_ptr=buf.data_ptr() + 5, shape=a.shape, bpl=2807), want, "device stride")
    assert np.array_equal(vb.dz_pyramid_level(None, 3, in_ptr=buf.data_ptr() + 5, shape=a.shape, bpl=2807), alpha_pyramid_levels(a)[3])
    wide = np.zeros((600, 800, 4), np.uint8)
    wide[:, :700] = a
    same_pyramid(vb.dzsave_png(wide[:, :700]), want, "host stride")
    vb.dzsave_png(a)
    pool = L.vb200_debug_dz_pool_used()
    try:
        # room for a few 256 x 256 tiles at a time: many batches, the same streams
        L.vb200_debug_dz_set_budget(24 << 20)
        same_pyramid(vb.dzsave_png(a), want, "small batches")
        assert L.vb200_debug_dz_pool_used() == pool
        L.vb200_debug_dz_set_budget(100000)
        cin, keep = vb._dz_image(a, None, None, None)
        handle = C.c_void_p(1)
        assert L.vb200_dzsave_png(C.byref(cin), None, None, C.byref(handle)) == -1 and handle.value is None
        assert b"more than the 100000 allowed" in L.vb200_error_buffer()
        L.vb200_error_clear()
        assert L.vb200_debug_dz_pool_used() == pool
    finally:
        L.vb200_debug_dz_set_budget(0)
    with pytest.raises(vb.Error, match="compression 2 is not built"):
        vb.dzsave_png(a, compression=2)
    same_pyramid(vb.dzsave_png(a), want, "again")
    assert L.vb200_debug_dz_pool_used() == pool
    # two calls at once from two host threads
    b = noise(500, 900, 2, 7)
    out, wants = {}, {"a": want, "b": vb.dzsave_png_host_twin(b, layout="zoomify", filter="paeth")}

    def run(key, image, kw):
        try:
            out[key] = vb.dzsave_png(image, **kw)
        except Exception as e:      # noqa: BLE001
            out[key] = e
    threads = [threading.Thread(target=run, args=("a", a, {})), threading.Thread(target=run, args=("b", b, {"layout": "zoomify", "filter": "paeth"}))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for key in ("a", "b"):
        assert not isinstance(out[key], Exception), out[key]
        same_pyramid(out[key], wants[key], "thread " + key)


@pytest.mark.gpu
def test_gpu_png_in_pyramid_out(vb):
    """RGBA PNG streams decoded on the device, the pyramid cut from the decoded frame where it lies"""
    import torch
    vb.init(0)
    a = rgba_photo(900, 1300, 3)
    b = io.BytesIO()
    PIL.fromarray(a).save(b, "PNG")
    stream = b.getvalue()
    w, h, bands = vb.png_geometry([stream])
    assert (w, h, bands) == (1300, 900, 4)
    frame = torch.empty((h, w, bands), dtype=torch.uint8, device="cuda")
    vb.png_decode_batch([stream], out_ptr=frame.data_ptr())
    got = vb.dzsave_png(None, "p", in_ptr=frame.data_ptr(), shape=(h, w, bands))
    same_pyramid(got, vb.dzsave_png_host_twin(np.asarray(PIL.open(io.BytesIO(stream))), "p"), "png in")

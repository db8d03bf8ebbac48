"""Deep Zoom / Zoomify tile pyramids (csrc/dzsave.cu) against vips_dzsave (foreign/dzsave.c).

Two statements of the same save are held against each other.  The library runs the whole-image one: each level is the 2 x 2
rounded mean of the level above, its last column / row read twice when its size is odd, and a tile is a clipped rect of its
level.  oracle/pydz.py restates the reference's strip walk loop for loop (strips of rows arriving, a line of tiles written
when a strip fills, the strip shrunk into the level below, overlap rows carried over, the flush at the bottom).  The sizes
below are chosen to take every branch of the walk: odd at some levels and even at others, a multiple of the tile step, one
more, one less.  Tile streams are libjpeg-turbo's (the one inside Pillow) byte for byte, as tests/test_jpeg_encode.py holds
the encoder's.

CPU tests run the kernels' per-pixel code and the encoder's host twin (vb200_debug_dzsave); -m gpu tests the kernels.
"""
import ctypes as C
import io
import os
import threading

import numpy as np
import pytest

PIL = pytest.importorskip("PIL.Image")

from test_jpeg import synth  # noqa: E402
from test_jpeg_encode import same_stream, turbo_encode  # noqa: E402

from oracle import pydz  # noqa: E402

SIZES = [1, 2, 3, 5, 253, 254, 255, 256, 257, 507, 508, 509, 510, 511, 512, 513, 1017]
TILES = [(254, 1), (256, 0), (128, 2), (16, 3), (17, 0), (7, 1)]
DEPTHS = ["onepixel", "onetile", "one"]
LAYOUTS = ["dz", "zoomify"]


@pytest.fixture(scope="module")
def vb():
    import libvips_b200 as vb
    vb.lib()
    return vb


def noise(h, w, bands, seed):
    a = np.random.default_rng(seed).integers(0, 256, (h, w, bands), dtype=np.uint8)
    return a


def pyramid_levels(a):
    """the whole-image statement in numpy, from the top: what the host twin and the kernels are held to"""
    out = [a]
    while out[-1].shape[0] > 1 or out[-1].shape[1] > 1:
        p = out[-1].astype(np.int32)
        if p.shape[0] & 1:
            p = np.concatenate([p, p[-1:]], 0)
        if p.shape[1] & 1:
            p = np.concatenate([p, p[:, -1:]], 1)
        out.append(((p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2] + 2) >> 2).astype(np.uint8))
    return out


def against_walk(vb, a, layout, tile_size, overlap, depth, strip_height=16):
    """the host twin's index, names, rects and side file, and the pixels its tiles are cut from, against the strip walk"""
    walk = pydz.dzsave(a, layout, tile_size, overlap, depth, "im", strip_height=strip_height)
    what = (a.shape, layout, tile_size, overlap, depth, strip_height)
    # entropy coding is tested on its own below: Q 1 keeps the streams of this grid small
    got = vb.dzsave_host_twin(a, "im", layout=layout, tile_size=tile_size, overlap=overlap, depth=depth, Q=1)
    assert [(n,) + g for n, g in enumerate(got.levels)] == walk.levels(), what
    top = len(got.levels) - 1
    levels = {}
    want = sorted(walk.tiles, key=lambda t: (t[1], t[3], t[2]))
    assert len(got.tiles) == len(want) == len(set(t[0] for t in want)), what
    for t, (name, n, x, y, rect, pixels) in zip(got.tiles, want):
        assert (t.name, t.level, t.x, t.y, t.rect) == (name, n, x, y, rect), what
        if n not in levels:
            levels[n] = vb.dz_pyramid_level_host_twin(a, top - n)
        left, tp, w, h = rect
        assert np.array_equal(levels[n][tp:tp + h, left:left + w], pixels), (what, name)
        assert t.bytes[:2] == b"\xff\xd8" and t.bytes[-2:] == b"\xff\xd9"
    assert got.sidecar == walk.sidecar(), what
    return got


def grid():
    """every width and every height of SIZES, and every one of the 2 x 6 x 3 x 2 option sets: each pairing of sizes takes the next
    two option sets with the large tiles, and each option set with the small tiles takes the next pairing of sizes up to 513 (they
    already make thousands of tiles there)"""
    options = [(b, t, d, l) for b in (1, 3) for t in TILES for d in DEPTHS for l in LAYOUTS]
    large, small = [o for o in options if o[1][0] >= 100], [o for o in options if o[1][0] < 100]
    cases, k = [], 0
    for i, w in enumerate(SIZES):
        for h in (SIZES[(5 * i + 3) % len(SIZES)], SIZES[(7 * i + 11) % len(SIZES)]):
            for _ in range(2):
                cases.append((w, h) + large[k % len(large)])
                k += 1
    some = SIZES[:-1]
    for j, o in enumerate(small):
        cases.append((some[(3 * j) % len(some)], some[(5 * j + 2) % len(some)]) + o)
    return cases


GRID = grid()


def test_grid_takes_every_option_set():
    assert {c[0] for c in GRID} == set(SIZES) == {c[1] for c in GRID}
    assert {c[3] for c in GRID} == set(TILES) and {(c[2], c[4], c[5]) for c in GRID} == {(b, d, l) for b in (1, 3) for d in DEPTHS for l in LAYOUTS}


@pytest.mark.parametrize("case", GRID, ids=lambda c: "%dx%dx%d-%d_%d-%s-%s" % (c[0], c[1], c[2], c[3][0], c[3][1], c[4], c[5]))
def test_strip_walk_is_the_whole_image_statement(vb, case):
    w, h, bands, (tile_size, overlap), depth, layout = case
    against_walk(vb, noise(h, w, bands, w * 31 + h), layout, tile_size, overlap, depth)


@pytest.mark.parametrize("strip_height", [1, 37])
def test_walk_does_not_depend_on_the_strip_height(vb, strip_height):
    for (w, h, bands, (tile_size, overlap), depth, layout) in GRID[::7]:
        against_walk(vb, noise(h, w, bands, w + h), layout, tile_size, overlap, depth, strip_height)


def test_flush_at_the_bottom(vb):
    """dzsave.c:1996-2011: a level one overlap taller than a multiple of the step gets its last line of tiles from strip_flush"""
    for h in (255, 509, 763):
        got = against_walk(vb, noise(h, 300, 3, h), "dz", None, None, None)
        assert got.levels[-1][3] == (h + 253) // 254 and got.tiles[-1].rect[3] == 2
    against_walk(vb, noise(45, 20, 1, 5), "zoomify", 16, 3, "one")      # step 13: rows 0, 13, 26, and 39 from the flush


def test_known_answers(vb):
    # pyramid_build :541-553 rounds up: 5 x 3 -> 3 x 2 -> 2 x 1 -> 1 x 1
    p = vb.dzsave_host_twin(noise(3, 5, 3, 1))
    assert [l[:2] for l in p.levels] == [(1, 1), (2, 1), (3, 2), (5, 3)]
    assert [t.name for t in p.tiles] == ["untitled_files/%d/0_0.jpeg" % n for n in range(4)]
    # 1000 x 700 with the defaults: 1000 -> 500 -> 250 -> 125 -> 63 -> 32 -> 16 -> 8 -> 4 -> 2 -> 1, so n = 0 .. 10
    p = vb.dzsave_host_twin(synth(700, 1000, seed=2), "photo")
    assert len(p.levels) == 11 and p.levels[10] == (1000, 700, 4, 3) and p.levels[9] == (500, 350, 2, 2) and p.levels[0] == (1, 1, 1, 1)
    top = {(t.x, t.y): t for t in p.tiles if t.level == 10}
    # image_strip_allocate :1139-1145: [x * 254 - 1, y * 254 - 1, 256, 256] clipped to 1000 x 700
    assert top[0, 0].rect == (0, 0, 255, 255) and top[1, 0].rect == (253, 0, 256, 255) and top[2, 0].rect == (507, 0, 256, 255)
    assert top[3, 0].rect == (761, 0, 239, 255) and top[1, 1].rect == (253, 253, 256, 256)
    assert top[0, 2].rect == (0, 507, 255, 193) and top[3, 2].rect == (761, 507, 239, 193)
    assert top[3, 2].name == "photo_files/10/3_2.jpeg"
    assert sum(l[2] * l[3] for l in p.levels) == len(p.tiles) == 12 + 4 + 9      # 4 x 3, 2 x 2, then one tile a level
    # write_dzi :596-608
    assert p.sidecar == ("photo.dzi", '<?xml version="1.0" encoding="UTF-8"?>\n<Image xmlns="http://schemas.microsoft.com/deepzoom/2008"\n'
                         '  Format="jpeg"\n  Overlap="1"\n  TileSize="254"\n  >\n  <Size \n    Height="700"\n    Width="1000"\n  />\n</Image>\n')
    # the reference drops a ".dz" left on the name (:2304-2310)
    assert vb.dzsave_host_twin(noise(3, 5, 3, 1), "a.b.dz").sidecar[0] == "a.b.dzi"


def test_zoomify_numbering(vb):
    # 40 x 24 tiles of 16 at the top: levels 640 x 384 (960 tiles), 320 x 192 (240), 160 x 96 (60), 80 x 48 (15), 40 x 24 (6), 20 x 12 (2),
    # 10 x 6 (1): onetile stops where the image fits one tile.  tile_name :1182-1193 counts the smaller levels first.
    p = vb.dzsave_host_twin(noise(384, 640, 1, 9), "z", layout="zoomify", tile_size=16, Q=1)
    assert [l[2] * l[3] for l in p.levels] == [1, 2, 6, 15, 60, 240, 960]
    names = {(t.level, t.x, t.y): t.name for t in p.tiles}
    assert names[0, 0, 0] == "z/TileGroup0/0-0-0.jpg"
    assert names[5, 11, 8] == "z/TileGroup0/5-11-8.jpg"        # 84 before the level + 8 * 20 + 11 = 255
    assert names[5, 12, 8] == "z/TileGroup1/5-12-8.jpg"        # 256: the first of the next group
    assert names[6, 39, 23] == "z/TileGroup5/6-39-23.jpg"      # 324 + 959 = 1283
    assert p.tiles[0].rect == (0, 0, 10, 6) and p.tiles[-1].rect == (624, 368, 16, 16)
    # write_properties :633-640
    assert p.sidecar == ("z/ImageProperties.xml",
                         '<IMAGE_PROPERTIES WIDTH="640" HEIGHT="384" NUMTILES="1284" NUMIMAGES="1" VERSION="1.8" TILESIZE="16" />\n')


def test_the_mean(vb):
    """region.c:1146-1149: (p00 + p01 + p10 + p11 + 2) >> 2, and level_generate_extras' repeated last column / row"""
    v = [0, 1, 2, 127, 128, 254, 255]
    quads = np.array([(a, b, c, d) for a in v for b in v for c in v for d in v], np.uint8)         # 2401 blocks of 2 x 2, side by side
    img = quads.reshape(-1, 2, 2).transpose(1, 0, 2).reshape(2, -1)
    got = vb.dz_pyramid_level_host_twin(img, 1)
    assert got.shape == (1, 2401, 1)
    assert np.array_equal(got[0, :, 0], (quads.astype(np.int32).sum(1) + 2) >> 2)
    # 3 x 3, by hand: the last column and row count twice
    a = np.array([[10, 20, 31], [40, 50, 61], [70, 81, 255]], np.uint8)
    want = [[(10 + 20 + 40 + 50 + 2) >> 2, (31 + 31 + 61 + 61 + 2) >> 2], [(70 + 81 + 70 + 81 + 2) >> 2, 255]]
    assert vb.dz_pyramid_level_host_twin(a, 1)[..., 0].tolist() == want
    # rounding happens at every level: three quarters that sum to 2 each round to 1, and 1 1 1 0 rounds to 1, where one 4 x 4 box
    # would round 6 / 16 to 0
    b = np.zeros((4, 4), np.uint8)
    b[0, :] = 1
    b[2, :2] = 1
    assert vb.dz_pyramid_level_host_twin(b, 1)[..., 0].tolist() == [[1, 1], [1, 0]] and vb.dz_pyramid_level_host_twin(b, 2)[0, 0, 0] == 1
    assert (int(b.sum()) + 8) >> 4 == 0
    for (h, w, bands) in ((7, 9, 3), (1, 6, 1), (6, 1, 3), (64, 65, 3), (129, 127, 1)):
        a = noise(h, w, bands, h * w)
        for n, want in enumerate(pyramid_levels(a)):
            assert np.array_equal(vb.dz_pyramid_level_host_twin(a, n), want), (h, w, bands, n)
    with pytest.raises(vb.Error, match="a 9 x 7 image has no level 5"):
        vb.dz_pyramid_level_host_twin(noise(7, 9, 3, 0), 5)


def pil_save(a, **kw):
    b = io.BytesIO()
    PIL.fromarray(a[..., 0] if a.shape[2] == 1 else a).save(b, "JPEG", **kw)
    return b.getvalue()


@pytest.mark.parametrize("shape", [(500, 600, 3), (200, 300, 1)], ids=["rgb", "grey"])
def test_tile_streams_are_libjpeg_turbos(vb, shape):
    a = synth(shape[0], shape[1], seed=shape[2], grey=shape[2] == 1).reshape(shape)
    walk = {t[0]: t[5] for t in pydz.dzsave(a, basename="t").tiles}
    p = vb.dzsave_host_twin(a, "t")
    shapes = {t.rect[2:] for t in p.tiles}
    assert {(1, 1), (2, 1), (3, 2)} <= shapes                  # the deep levels: a pixel, a row of two ...
    for t in p.tiles:
        pix = walk[t.name]
        same_stream(t.bytes, turbo_encode(pix[..., 0] if shape[2] == 1 else pix, 75, 2 if shape[2] == 3 else 0), t.name)
    # a column and a row of pixels as tiles
    for thin in (a[:, :1], a[:1, :]):
        for t, (name, _, _, _, _, pix) in zip(vb.dzsave_host_twin(thin, depth="one").tiles, pydz.dzsave(thin, depth="one").tiles):
            assert 1 in t.rect[2:] and t.rect[2:] == pix.shape[1::-1] and t.name == name
            same_stream(t.bytes, turbo_encode(pix[..., 0] if shape[2] == 1 else pix, 75, 2 if shape[2] == 3 else 0), name)
    # vips_jpegsave's options reach every tile: Q 90 stops subsampling (vips2jpeg.c:676-690)
    for kw, pil in (({"Q": 90}, {"quality": 90, "subsampling": 0}), ({"optimize_coding": True}, {"quality": 75, "subsampling": 2, "optimize": True}),
                    ({"interlace": True}, {"quality": 75, "subsampling": 2, "progressive": True})):
        if shape[2] == 1:
            pil["subsampling"] = 0
        for t in vb.dzsave_host_twin(a, "t", **kw).tiles:
            assert t.bytes == pil_save(walk[t.name], **pil), (kw, t.name)


def test_declines(vb):
    a = noise(40, 30, 3, 0)
    refused = [({"layout": "google"}, "layout google not supported on the device path"),
               ({"layout": "iiif"}, "layout iiif not supported on the device path"),
               ({"layout": "iiif3"}, "layout iiif3 not supported on the device path"),
               ({"region_shrink": "median"}, "region_shrink other than mean not supported on the device path"),
               ({"region_shrink": "nearest"}, "region_shrink other than mean not supported on the device path"),
               ({"skip_blanks": 0}, "skip_blanks not supported on the device path"),
               ({"skip_blanks": 5}, "skip_blanks not supported on the device path"),
               ({"container": "zip"}, "zip containers not supported on the device path"),
               ({"container": "szi"}, "zip containers not supported on the device path"),
               ({"suffix": ".png"}, r"suffix \.png not supported on the device path"),
               ({"suffix": ".webp"}, r"suffix \.webp not supported on the device path"),
               ({"suffix": ".jpg[Q=90]"}, "suffix options not supported on the device path"),
               ({"layout": "zoomify", "tile_size": 16, "overlap": 9}, "overlap above half the tile size is not supported on the device path"),
               ({"layout": "zoomify", "tile_size": 16, "overlap": 16}, "dzsave: overlap too large"),
               ({"layout": "zoomify", "tile_size": 16, "overlap": 20}, "dzsave: overlap too large"),
               ({"restart_interval": 70000}, "restart_interval 70000 outside")]
    for kw, message in refused:
        with pytest.raises(vb.Error, match=message):
            vb.dzsave_host_twin(a, **kw)
    for bad, message in ((noise(8, 8, 2, 0), "2-band images not supported on the device path"),
                         (noise(8, 8, 4, 0), "4-band images not supported on the device path"),
                         (noise(8, 8, 3, 0).astype(np.uint16), "band format 2 not supported on the device path"),
                         (noise(8, 8, 1, 0).astype(np.float32), "band format 6 not supported on the device path")):
        with pytest.raises(vb.Error, match=message):
            vb.dzsave_host_twin(bad)
    # a failed save hands nothing back
    L = vb.lib()
    cin, keep = vb._dz_image(noise(8, 8, 2, 0), None, None, None)
    handle = C.c_void_p(1)
    assert L.vb200_debug_dzsave(C.byref(cin), None, C.byref(handle)) == -1 and handle.value is None
    L.vb200_error_clear()
    # in the dz layout an overlap as wide as the tile is legal (the step is the tile size)
    assert len(vb.dzsave_host_twin(a, tile_size=16, overlap=16, Q=1).tiles) > 6
    # ".JPG" is a JPEG suffix too
    assert vb.dzsave_host_twin(a, suffix=".JPG").tiles[0].name == "untitled_files/0/0_0.JPG"


def test_write_makes_the_tree_a_viewer_reads(vb, tmp_path):
    a = synth(300, 520, seed=4)
    vb.dzsave_host_twin(a, "slide").write(str(tmp_path))
    assert sorted(os.listdir(tmp_path)) == ["slide.dzi", "slide_files"]
    assert sorted(os.listdir(tmp_path / "slide_files"), key=int) == [str(n) for n in range(11)]
    assert sorted(os.listdir(tmp_path / "slide_files" / "10")) == ["0_0.jpeg", "0_1.jpeg", "1_0.jpeg", "1_1.jpeg", "2_0.jpeg", "2_1.jpeg"]
    assert 'Width="520"' in (tmp_path / "slide.dzi").read_text()
    assert PIL.open(tmp_path / "slide_files" / "10" / "2_1.jpeg").size == (520 - 507, 300 - 253)
    assert PIL.open(tmp_path / "slide_files" / "0" / "0_0.jpeg").size == (1, 1)
    vb.dzsave_host_twin(a, "slide", layout="zoomify").write(str(tmp_path / "z"))
    assert sorted(os.listdir(tmp_path / "z" / "slide")) == ["ImageProperties.xml", "TileGroup0"]
    assert sorted(os.listdir(tmp_path / "z" / "slide" / "TileGroup0")) == ["0-0-0.jpg", "1-0-0.jpg", "1-1-0.jpg", "2-0-0.jpg", "2-0-1.jpg", "2-1-0.jpg",
                                                                           "2-1-1.jpg", "2-2-0.jpg", "2-2-1.jpg"]


def test_abi(vb):
    """VB200DzOptions as include/vb200.h lays it out: seven ints, the suffix pointer, VB200JpegSaveOptions"""
    assert C.sizeof(vb.DzOptions) == 64 and vb.DzOptions.suffix.offset == 32 and vb.DzOptions.jpeg.offset == 40
    assert C.sizeof(vb.JpegSaveOptions) == 20
    L = C.CDLL(vb.library_path())
    for name in ("vb200_dzsave", "vb200_debug_dzsave", "vb200_dz_free", "vb200_dz_levels", "vb200_dz_level_geometry", "vb200_dz_tiles", "vb200_dz_tile",
                 "vb200_dz_tile_name", "vb200_dz_sidecar", "vb200_dz_pyramid_level", "vb200_debug_dz_pyramid_level", "vb200_debug_dz_set_budget",
                 "vb200_debug_dz_pool_used", "vb200_debug_dz_times"):
        assert hasattr(L, name), name
    # options NULL is every default; a short name buffer is an error, not an overrun
    cin, keep = vb._dz_image(noise(8, 8, 3, 0), None, None, None)
    handle = C.c_void_p()
    assert vb.lib().vb200_debug_dzsave(C.byref(cin), None, C.byref(handle)) == 0
    small = C.create_string_buffer(8)
    assert vb.lib().vb200_dz_tile_name(handle, 0, None, small, len(small)) == -1
    assert vb.lib().vb200_dz_tile(handle, 99, *([None] * 9)) == -1
    vb.lib().vb200_error_clear()
    vb.lib().vb200_dz_free(handle)


# ------------------------------------------------------------------ GPU

def same_pyramid(got, want, what):
    assert got.levels == want.levels and got.sidecar == want.sidecar, what
    assert len(got.tiles) == len(want.tiles), what
    for g, w in zip(got.tiles, want.tiles):
        assert (g.name, g.level, g.x, g.y, g.rect) == (w.name, w.level, w.x, w.y, w.rect), what
        assert g.bytes == w.bytes, (what, g.name)


def decodes_to(vb, p, a, what):
    """the sanity net: every tile decodes to its own size, and at the full-size level (the deeper ones of the test image shrink
    to noise, which Q 75 with halved chroma does not keep) to within JPEG error of the pixels it was cut from"""
    top = len(p.levels) - 1
    for t in p.tiles:
        left, tp, w, h = t.rect
        got = np.asarray(PIL.open(io.BytesIO(t.bytes)))
        assert got.shape[:2] == (h, w), (what, t.name)
        if t.level == top:
            want = a[tp:tp + h, left:left + w].astype(np.int32)
            assert np.abs(got.reshape(want.shape).astype(np.int32) - want).mean() < 12, (what, t.name)


@pytest.mark.gpu
def test_gpu_equals_the_host_twin(vb):
    import torch
    vb.init(0)
    for (w, h, bands, (tile_size, overlap), depth, layout) in GRID[::5] + [(4096, 4096, 3, (None, None), None, "dz"), (5000, 3000, 3, (None, None), None, "dz"),
                                                                          (2000, 1500, 1, (None, None), None, "zoomify")]:
        a = synth(h, w, seed=w + h, grey=bands == 1).reshape(h, w, bands)
        kw = dict(layout=layout, tile_size=tile_size, overlap=overlap, depth=depth)
        want = vb.dzsave_host_twin(a, "g", **kw)
        same_pyramid(vb.dzsave(a, "g", **kw), want, ("host", w, h, kw))
        d = torch.from_numpy(a).cuda()
        same_pyramid(vb.dzsave(None, "g", in_ptr=d.data_ptr(), shape=a.shape, **kw), want, ("device", w, h, kw))
        if max(w, h) >= 2000:
            decodes_to(vb, want, a, (w, h))
    a = synth(300, 400, seed=1)
    for kw in ({"Q": 92}, {"optimize_coding": True}, {"interlace": True}, {"restart_interval": 3}, {"subsample_mode": "off"}):
        same_pyramid(vb.dzsave(a, **kw), vb.dzsave_host_twin(a, **kw), kw)
    same_pyramid(vb.Image(a).dzsave("im", layout="zoomify"), vb.dzsave_host_twin(a, "im", layout="zoomify"), "Image.dzsave")


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(4097, 4095, 3), (1, 4096, 1), (4096, 1, 3), (65537, 3, 1), (3, 65537, 3)], ids=lambda s: "%dx%dx%d" % s)
def test_gpu_pyramid_levels(vb, size):
    import torch
    vb.init(0)
    w, h, bands = size
    a = noise(h, w, bands, w + h)
    d = torch.from_numpy(a).cuda()
    for n, want in enumerate(pyramid_levels(a)):
        assert np.array_equal(vb.dz_pyramid_level(None, n, in_ptr=d.data_ptr(), shape=a.shape), want), (size, n)
        if n % 3 == 1:
            assert np.array_equal(vb.dz_pyramid_level(a, n), want), (size, n, "host")
            assert np.array_equal(vb.dz_pyramid_level_host_twin(a, n), want), (size, n, "twin")


@pytest.mark.gpu
def test_gpu_strides_alignment_and_threads(vb):
    import torch
    vb.init(0)
    a = synth(600, 700, seed=6)
    want = vb.dzsave_host_twin(a)
    # rows 2113 bytes apart, the first pixel 5 bytes into the allocation: no 16-byte load is legal
    buf = torch.zeros(5 + 600 * 2113, dtype=torch.uint8, device="cuda")
    buf[5:].view(600, 2113)[:, :2100] = torch.from_numpy(a.reshape(600, 2100)).cuda()
    same_pyramid(vb.dzsave(None, in_ptr=buf.data_ptr() + 5, shape=a.shape, bpl=2113), want, "device stride")
    assert np.array_equal(vb.dz_pyramid_level(None, 3, in_ptr=buf.data_ptr() + 5, shape=a.shape, bpl=2113), pyramid_levels(a)[3])
    wide = np.zeros((600, 800, 3), np.uint8)
    wide[:, :700] = a
    same_pyramid(vb.dzsave(wide[:, :700]), want, "host stride")
    # two calls at once from two host threads
    b = synth(500, 900, seed=7)
    out, wants = {}, {"a": want, "b": vb.dzsave_host_twin(b, layout="zoomify")}

    def run(key, image, kw):
        try:
            out[key] = vb.dzsave(image, **kw)
        except Exception as e:      # noqa: BLE001
            out[key] = e
    threads = [threading.Thread(target=run, args=("a", a, {})), threading.Thread(target=run, args=("b", b, {"layout": "zoomify"}))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for key in ("a", "b"):
        assert not isinstance(out[key], Exception), out[key]
        same_pyramid(out[key], wants[key], "thread " + key)


@pytest.mark.gpu
def test_gpu_jpeg_in_pyramid_out(vb):
    """decode on the device, cut the pyramid from the decoded frame where it lies"""
    import torch
    from test_jpeg import encode, turbo_decode
    vb.init(0)
    stream = encode(synth(900, 1300, seed=3), 90, 2)
    w, h, bands = vb.jpeg_geometry([stream])
    frame = torch.empty((h, w, bands), dtype=torch.uint8, device="cuda")
    vb.jpeg_decode_batch([stream], out_ptr=frame.data_ptr())
    got = vb.dzsave(None, "p", in_ptr=frame.data_ptr(), shape=(h, w, bands))
    same_pyramid(got, vb.dzsave_host_twin(turbo_decode(stream, 1), "p"), "jpeg in")


@pytest.mark.gpu
def test_gpu_leaves_nothing_allocated(vb):
    vb.init(0)
    L = vb.lib()
    a = synth(700, 900, seed=8)
    want = vb.dzsave_host_twin(a)
    vb.dzsave(a)
    before = L.vb200_debug_dz_pool_used()
    same_pyramid(vb.dzsave(a), want, "again")
    assert L.vb200_debug_dz_pool_used() == before
    try:
        # room for three 256 x 256 tiles at a time: the tiles of the top level take several batches, same streams
        L.vb200_debug_dz_set_budget(4 << 20)
        same_pyramid(vb.dzsave(a), want, "small batches")
        assert L.vb200_debug_dz_pool_used() == before
        # no room for one tile: an error, no pyramid, nothing left on the device
        L.vb200_debug_dz_set_budget(100000)
        cin, keep = vb._dz_image(a, None, None, None)
        handle = C.c_void_p(1)
        assert L.vb200_dzsave(C.byref(cin), None, C.byref(handle)) == -1 and handle.value is None
        assert b"more than the 100000 allowed" in L.vb200_error_buffer()
        L.vb200_error_clear()
        assert L.vb200_debug_dz_pool_used() == before
    finally:
        L.vb200_debug_dz_set_budget(0)
    with pytest.raises(vb.Error, match="layout google not supported"):
        vb.dzsave(a, layout="google")
    assert L.vb200_debug_dz_pool_used() == before

"""Thumbnails of page strips (multi-page images stacked vertically with libvips' "page-height"): vips_thumbnail's
page-height shrink (thumbnail.c:825-839), premultiply rule (:848-861) and output page height (:904-917), through
vb200_thumbnail_image_pages, plans made with vb200_thumbnail_plan_new_pages, vb200_thumbnail_plan_run_gif_pages and
vb200_thumbnail_buffer_pages.

The rules are restated here around the oracle's own resize (page_shrink / orc_page_thumbnail) and, for the reference,
around its own vips_thumbnail_calculate_shrink and vips_resize (ref_pages_size_table / ref_page_thumbnail).  Those two keep
their answers in a file of their own, tests/golden/ref_results_pages.json.gz, keyed and encoded as pyref keys and encodes
its answers, so that runs without the reference build still check them; run with oracle/_ref built and VB200_REF_RECORD=1
to record them again.
"""
import atexit
import ctypes as C
import functools
import gzip
import json
import os

import numpy as np
import pytest

import libvips_b200 as vb
from oracle import pyoracle, pyref

GOLDEN_GIF = os.path.join(os.path.dirname(__file__), "golden", "gif")
PAGES_GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ref_results_pages.json.gz")
_PAGES_NEW = {}


def _save_pages_answers():
    old = {}
    if os.path.exists(PAGES_GOLDEN):
        with gzip.open(PAGES_GOLDEN, "rt") as f:
            old = json.load(f)
    old.update(_PAGES_NEW)
    with gzip.GzipFile(PAGES_GOLDEN, "wb", mtime=0) as f:
        f.write(json.dumps(old, sort_keys=True, separators=(",", ":")).encode())


def recorded_pages(fn):
    """pyref.recorded, with the answers in PAGES_GOLDEN: computed by the reference library when it is built (its own
    recorded calls inside fn are not recorded separately), read from PAGES_GOLDEN otherwise"""
    @functools.wraps(fn)
    def wrap(*args, **kw):
        key = pyref._key(fn.__qualname__, args, kw)
        if pyref.live():
            depth = getattr(pyref._DEPTH, "n", 0)
            pyref._DEPTH.n = depth + 1
            try:
                v = fn(*args, **kw)
            finally:
                pyref._DEPTH.n = depth
            if os.environ.get("VB200_REF_RECORD"):
                if not _PAGES_NEW:
                    atexit.register(_save_pages_answers)
                _PAGES_NEW[key] = pyref._encode(v)
            return v
        with gzip.open(PAGES_GOLDEN, "rt") as f:
            answers = json.load(f)
        if key not in answers:
            raise KeyError("no recorded reference answer for this call (%s); record it with oracle/_ref built and "
                           "VB200_REF_RECORD=1" % key)
        return pyref._decode(answers[key])
    return wrap


def ref_available():
    return pyref.live() or os.path.exists(PAGES_GOLDEN)


# ------------------------------------------------------------------------------------------------ the rules, restated

def n_loaded_pages(height, page_height):
    """vips_image_get_page_height (header.c:889-901) -> (page height, pages)"""
    ph = page_height if page_height and 0 < page_height < height and height % page_height == 0 else height
    return ph, height // ph


def orc_shrink(w, h, tw, th, size):
    """the oracle's vips_thumbnail_calculate_shrink (orc_thumbnail_size sets the shrinks before it sizes the resize, which
    fails for mixed up / down shrinks)"""
    hs, vs, ow, oh = C.c_double(), C.c_double(), C.c_int(), C.c_int()
    pyoracle.lib().orc_thumbnail_size(w, h, tw, th, pyoracle.SIZES[size], C.byref(hs), C.byref(vs), C.byref(ow), C.byref(oh))
    return hs.value, vs.value


def page_shrink(w, ph, n, tw, th, size, calculate_shrink):
    """thumbnail.c:825-839: the shrink of one page, then vshrink so that every page lands on whole rows"""
    hs, vs = calculate_shrink(w, ph, tw, th, size)
    if n > 1:
        target_page_height = int(np.rint(ph / vs))  # rint: half to even
        vs = (ph * n) / (target_page_height * n)
    return hs, vs


def resize_size(w, h, hs, vs):
    ow, oh = C.c_int(), C.c_int()
    if pyoracle.lib().orc_resize_size(w, h, C.c_double(1.0 / hs), C.c_double(1.0 / vs), pyoracle.KERNELS["lanczos3"], C.c_double(2.0),
                                      C.byref(ow), C.byref(oh)):
        raise ValueError("resize size")
    return ow.value, oh.value


def pages_size(w, ph, n, tw, th, size, calculate_shrink=orc_shrink):
    """(hshrink, vshrink, out_width, out_height, out_page_height), or None where the device declines a single page too
    (one shrink up and the other down)"""
    hs, vs = page_shrink(w, ph, n, tw, th, size, calculate_shrink)
    if (hs < 1 or vs < 1) and (hs > 1 or vs > 1):
        return None
    ow, oh = resize_size(w, ph * n, hs, vs)
    oph = oh
    if n > 1:
        oph = int(np.rint(ph / vs))  # thumbnail.c:904-917, read back as vips_image_get_page_height does
        if not (0 < oph < oh and oh % oph == 0):
            oph = oh
    return hs, vs, ow, oh, oph


def size_table(cases, fn):
    rows = []
    for c in cases:
        r = fn(*c)
        rows.append(r if r is not None else (-1.0,) * 5)
    return np.array(rows, np.float64)


@recorded_pages
def ref_pages_size_table(cases):
    """pages_size over cases, built on the reference's own vips_thumbnail_calculate_shrink (ref_shim)"""
    return size_table(cases, lambda *c: pages_size(*c, calculate_shrink=pyref.thumbnail_calculate_shrink))


def orc_page_thumbnail(a, page_height, tw, th=None, size="both", linear=False):
    """vips_thumbnail_image of a strip, the oracle's premultiply / resize / unpremultiply (linear: through scRGB, as
    orc_thumbnail_image_linear) with the page rules -> (pixels, page height of the result or None)"""
    H, W, b = a.shape
    ph, n = n_loaded_pages(H, page_height)
    th = th or tw
    hs, vs = page_shrink(W, ph, n, tw, th, size, orc_shrink)
    premul = (b == 2 or b >= 4) and hs != 1.0 and vs != 1.0
    if linear:
        x = pyoracle.colourspace(a, "scrgb", "srgb")
        if premul:
            x = pyoracle.premultiply(x, 1.0)
        x = pyoracle.resize(x, 1.0 / hs, 1.0 / vs)
        if premul:
            x = pyoracle.unpremultiply(x, 1.0)
        x = pyoracle.colourspace(x, "srgb", "scrgb")
    else:
        x = pyoracle.premultiply(a, 255.0, uchar=True) if premul else a
        x = pyoracle.resize(x, 1.0 / hs, 1.0 / vs)
        if premul:
            x = pyoracle.unpremultiply(x, 255.0, uchar=True)
    oph = pages_size(W, ph, n, tw, th, size)[4]
    return x, (oph if oph < x.shape[0] else None)


@recorded_pages
def ref_page_thumbnail(a, page_height, tw, th, size):
    """the reference's premultiply / vips_resize / unpremultiply over the strip, with the page rules"""
    H, W, b = a.shape
    ph, n = n_loaded_pages(H, page_height)
    hs, vs = page_shrink(W, ph, n, tw, th, size, pyref.thumbnail_calculate_shrink)
    im = pyref.RefImage.from_array(a)
    premul = (b == 2 or b >= 4) and hs != 1.0 and vs != 1.0
    if premul:
        im = im.premultiply(uchar=True)
    im = im.resize(1.0 / hs, 1.0 / vs)
    if premul:
        im = im.unpremultiply(uchar=True)
    return im.numpy()


# ------------------------------------------------------------------------------------------------ CPU: size arithmetic

SIZES = ("both", "up", "down", "force")
TARGETS = ((25, 25), (25, 30), (7, 7), (100, 100))


def sweep_cases():
    return [(w, ph, n, tw, th, size) for w in range(1, 65) for ph in range(1, 65) for n in (2, 3, 7) for (tw, th) in TARGETS
            for size in SIZES]


@pytest.fixture(scope="module")
def sweep():
    cases = sweep_cases()
    return cases, size_table(cases, vb.thumbnail_pages_size)


def test_size_sweep_against_the_restatement(sweep):
    cases, got = sweep
    want = size_table(cases, pages_size)
    bad = np.nonzero((got != want).any(axis=1))[0]
    assert bad.size == 0, [(cases[i], got[i], want[i]) for i in bad[:5]]
    # the sweep reaches every branch
    hs, vs = got[:, 0], got[:, 1]
    assert (got[:, 0] == -1).any(), "mixed up / down strips"
    assert ((hs > 0) & (hs < 1) & (vs < 1)).any(), "enlarging strips"
    assert ((hs == 1) & (vs != 1) & (vs > 0)).any(), "hshrink 1, vshrink not"
    assert ((got[:, 4] != got[:, 3]) & (got[:, 4] > 0)).any(), "a page height on the result"


def test_size_sweep_against_the_reference(sweep):
    if not ref_available():
        pytest.skip("no reference build and no recorded answers")
    cases, got = sweep
    want = ref_pages_size_table(cases)
    assert np.array_equal(got, want), pyref.difference(got, want)


def test_size_known_answers():
    # rint(25 / 2) = 12.5 -> 12 (half to even), so vshrink = 50 / 24 = 25 / 12
    assert vb.thumbnail_pages_size(50, 25, 2, 25) == (2.0, 25 / 12, 25, 24, 12)
    # force: hshrink 1 with vshrink 64 / 30 -> every page 30 rows
    hs, vs, ow, oh, oph = vb.thumbnail_pages_size(25, 64, 3, 25, 30, "force")
    assert (hs, ow, oh, oph) == (1.0, 25, 90, 30) and vs == 192 / 90
    # an enlarging strip: 5-row pages to 20 rows
    assert vb.thumbnail_pages_size(10, 5, 3, 40) == (0.25, 0.25, 40, 60, 20)
    # up on one axis, down on the other: declined, as for one page
    assert vb.thumbnail_pages_size(10, 5, 3, 40, 3, "force") is None


@pytest.mark.parametrize("w,h,tw,th,size", [(1024, 768, 128, 0, "both"), (50, 50, 25, 0, "both"), (640, 480, 800, 0, "up"),
                                            (333, 555, 100, 50, "force"), (7, 3, 1, 0, "down"), (4000, 3000, 200, 0, "both")])
def test_one_page_is_todays_plan(w, h, tw, th, size):
    hs, vs, ow, oh = pyoracle.thumbnail_size(w, h, tw, th or tw, size)
    assert vb.thumbnail_pages_size(w, h, 1, tw, th, size) == (hs, vs, ow, oh, oh)
    for bands in (1, 3, 4):
        name = C.create_string_buffer(256)
        assert vb.lib().vb200_debug_thumbnail_kernel(w, h, bands, int(bands == 4), tw, th, vb.SIZES[size], name, 256) == 0
        assert vb.thumbnail_pages_kernel(w, h, 1, bands, tw, th, size) == name.value.decode()


def test_strips_pick_fused_kernels():
    for case in ((320, 240, 16, 4, 128), (480, 270, 100, 3, 200), (50, 25, 2, 4, 25), (64, 70, 1000, 4, 16)):
        k = vb.thumbnail_pages_kernel(*case)
        assert k and k.startswith("thumbnail_fused"), (case, k)


def test_strip_limit():
    assert vb.thumbnail_pages_kernel(16384, 16383, 2, 4, 128) is not None
    assert vb.thumbnail_pages_kernel(16384, 16384, 2, 4, 128) is None  # 2^31 bytes


def strip(seed, W, ph, n, bands):
    return np.random.default_rng(seed).integers(0, 256, (ph * n, W, bands), dtype=np.uint8)


def test_restatement_is_the_single_page_oracle():
    rng = np.random.default_rng(3)
    for (h, w, b, tw, size) in ((61, 47, 4, 20, "both"), (40, 33, 3, 90, "both"), (29, 31, 2, 9, "force"), (50, 50, 4, 25, "down")):
        a = rng.integers(0, 256, (h, w, b), dtype=np.uint8)
        assert np.array_equal(orc_page_thumbnail(a, None, tw, None, size)[0], pyoracle.thumbnail_image(a, tw, size=size))
        if b >= 3 and size != "force" and tw < w:
            assert np.array_equal(orc_page_thumbnail(a, None, tw, None, size, linear=True)[0],
                                  pyoracle.thumbnail_image(a, tw, size=size, linear=True))


# page heights where shrinkv boxes and reducev windows straddle the page seams; 1-4 bands, with and without alpha
PIN_CASES = [(37, 23, 3, 1, 10, None, "both"), (41, 19, 4, 2, 11, None, "both"), (50, 25, 2, 3, 25, None, "both"),
             (64, 17, 4, 4, 9, 9, "force"), (30, 13, 5, 4, 7, None, "both"), (16, 9, 3, 4, 40, None, "both"),
             (25, 64, 3, 4, 25, 30, "force"), (33, 31, 3, 4, 5, None, "both")]


@pytest.mark.parametrize("case", PIN_CASES, ids=lambda c: "%dx%dx%d-%db-%s" % (c[0], c[1], c[2], c[3], c[6]))
def test_oracle_pinned_to_the_reference(case):
    if not ref_available():
        pytest.skip("no reference build and no recorded answers")
    W, ph, n, bands, tw, th, size = case
    a = strip(sum(case[:5]), W, ph, n, bands)
    got = orc_page_thumbnail(a, ph, tw, th, size)[0]
    want = ref_page_thumbnail(a, ph, tw, th or tw, size)
    assert np.array_equal(got, want), pyref.difference(got, want)


# ------------------------------------------------------------------------------------------------ on the device

# (W, page height, pages, bands, target width, target height, size)
GPU_CASES = PIN_CASES + [(320, 240, 16, 4, 128, None, "both"), (480, 270, 10, 3, 200, None, "both"),
                         (64, 70, 1000, 4, 16, None, "both"),    # 70 000 rows
                         (1024, 1024, 17, 4, 200, None, "both")]  # 68 MiB: more than one slice of the host pump


def gpu_id(c):
    W, ph, n, bands, tw, th, size = c
    return "%dx%dx%d-%db-%d-%s-%s" % (W, ph, n, bands, tw, size, vb.thumbnail_pages_kernel(W, ph, n, bands, tw, th, size))


@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_CASES, ids=gpu_id)
def test_gpu_image_pages_and_plans(vb, case):
    import torch
    W, ph, n, bands, tw, th, size = case
    a = strip(sum(case[:5]), W, ph, n, bands)
    want, want_ph = orc_page_thumbnail(a, ph, tw, th, size)
    got = vb.Image(a, page_height=ph).thumbnail_image(tw, th, size)
    assert np.array_equal(got.numpy(), want)
    assert got.page_height == want_ph
    plan = vb.ThumbnailPlan(W, ph * n, bands, tw, th, size, page_height=ph)
    assert plan.kernel == vb.thumbnail_pages_kernel(W, ph, n, bands, tw, th, size)
    assert (plan.out_height, plan.out_width, plan.out_page_height) == (want.shape[0], want.shape[1], want_ph)
    frames = np.stack([a, a[::-1].copy()])
    want2 = orc_page_thumbnail(frames[1], ph, tw, th, size)[0]
    got = plan.run_host(frames)
    assert np.array_equal(got[0], want) and np.array_equal(got[1], want2)
    din = torch.from_numpy(frames).cuda()
    dout = torch.empty((2,) + want.shape, dtype=torch.uint8, device="cuda")
    plan.run_device(din.data_ptr(), dout.data_ptr(), 2)
    torch.cuda.synchronize()
    assert np.array_equal(dout.cpu().numpy(), got)
    plan.close()


@pytest.mark.gpu
def test_gpu_image_pages_icc_and_linear(vb):
    from icc_fixtures import rgb_profile
    prof = bytes(rgb_profile("srgb"))
    for bands in (3, 4):
        # 64-row pages at shrink 4: the page rules keep vshrink = hshrink, so the single-image entries on the same strip,
        # with a target height that leaves the width in charge, compute the same thumbnail
        a = strip(bands, 200, 64, 3, bands)
        page = vb.Image(a, page_height=64)
        whole = vb.Image(a)
        assert np.array_equal(page.thumbnail_image(50).numpy(), orc_page_thumbnail(a, 64, 50)[0])
        assert np.array_equal(page.thumbnail_image(50).numpy(), whole.thumbnail_image(50, 10 ** 6).numpy())
        got = page.thumbnail_image(50, output_profile=prof)
        assert got.page_height == 16
        assert np.array_equal(got.numpy(), whole.thumbnail_image(50, 10 ** 6, output_profile=prof).numpy())
        assert np.array_equal(page.thumbnail_image_linear(50, output_profile=prof).numpy(),
                              whole.thumbnail_image_linear(50, 10 ** 6, output_profile=prof).numpy())
        assert np.array_equal(page.thumbnail_image_linear(50).numpy(), whole.thumbnail_image_linear(50, 10 ** 6).numpy())
        # linear without profiles where vshrink is adjusted (rint(25 / 2) = 12): against the oracle's linear chain
        b = strip(bands + 10, 50, 25, 3, bands)
        got = vb.Image(b, page_height=25).thumbnail_image(25, linear=True)
        want, want_ph = orc_page_thumbnail(b, 25, 25, linear=True)
        assert np.array_equal(got.numpy(), want) and got.page_height == want_ph == 12
        assert np.array_equal(vb.Image(b, page_height=25).thumbnail_image_linear(25).numpy(), want)


def gif_fixture(name):
    with open(os.path.join(GOLDEN_GIF, name + ".gif"), "rb") as f:
        return f.read()


def gif_streams():
    from test_gif import animated
    rng = np.random.default_rng(31)
    out = {name: gif_fixture(name) for name in ("cogs", "cramps", "dispose-background", "dispose-previous")}
    out["writer-rgba"] = animated(rng, 97, 61, 6)
    out["writer-rgb"] = animated(rng, 64, 48, 4, trans=False)
    return out


@pytest.mark.gpu
def test_gpu_gif_pages(vb):
    for name, s in gif_streams().items():
        w, sh, bands, frames = vb.gif_geometry(s)
        for page, n in {(0, -1), (0, 1), (frames // 2, -1), (frames // 2, 1), (max(0, frames - 3), min(2, frames))}:
            dec = vb.gif_decode_host_twin(s, page, n)
            pages = dec.shape[0] // sh
            for tw in (32, 150):
                want, want_ph = orc_page_thumbnail(dec, sh if pages > 1 else None, tw)
                got, got_ph = vb.thumbnail_buffer(s, tw, page=page, n=n, return_page_height=True)
                assert np.array_equal(got, want), (name, page, n, tw)
                assert got_ph == want_ph, (name, page, n, tw)
                plan = vb.ThumbnailPlan(w, dec.shape[0], dec.shape[2], tw, page_height=sh if pages > 1 else None)
                assert plan.out_page_height == want_ph
                got = plan.run_gif([s, s], page=page, n=n)
                plan.close()
                assert np.array_equal(got[0], want) and np.array_equal(got[1], want), (name, page, n, tw)
            got = vb.thumbnail_buffer_linear(s, 40, page=page, n=n)
            assert np.array_equal(got, orc_page_thumbnail(dec, sh if pages > 1 else None, 40, linear=True)[0]), (name, page, n)
        # gifload_buffer(n = -1) carries the page height into thumbnail_image
        im = vb.Image.gifload_buffer(s, 0, -1)
        assert im.page_height == (sh if frames > 1 else None)
        assert np.array_equal(im.thumbnail_image(32).numpy(), vb.thumbnail_buffer(s, 32, n=-1))


@pytest.mark.gpu
def test_gpu_declines(vb):
    import io
    from PIL import Image as PIL
    a = np.random.default_rng(2).integers(0, 256, (40, 50, 3), dtype=np.uint8)
    for fmt, loader in (("JPEG", "jpegload"), ("PNG", "pngload")):
        buf = io.BytesIO()
        PIL.fromarray(a).save(buf, fmt)
        s = buf.getvalue()
        for page, n in ((0, -1), (1, 1), (0, 2)):
            with pytest.raises(vb.Error, match="%s has no page or n option" % loader):
                vb.thumbnail_buffer(s, 20, page=page, n=n)
        assert np.array_equal(vb.thumbnail_buffer(s, 20, return_page_height=True)[0], vb.thumbnail_buffer(s, 20))
    # a batch of streams with different page counts writes nothing
    from test_gif import animated
    rng = np.random.default_rng(8)
    s4, s5 = animated(rng, 40, 30, 4), animated(rng, 40, 30, 5)
    plan = vb.ThumbnailPlan(40, 120, 4, 20, page_height=30)
    b = vb.StreamBatch([s4, s5])
    out = np.full((2, plan.out_height, plan.out_width, 4), 77, np.uint8)
    rc = vb.lib().vb200_thumbnail_plan_run_gif_pages(plan._p, b.ptrs, b.lens, 2, 0, -1, out.ctypes.data_as(C.c_void_p), vb.HOST,
                                                     plan.out_frame_bytes)
    assert rc == -1 and "one geometry" in vb.lib().vb200_error_buffer().decode()
    vb.lib().vb200_error_clear()
    assert (out == 77).all()
    # a plan whose pages are not the screen's
    with pytest.raises(vb.Error, match="pages of 40 rows"):
        vb.ThumbnailPlan(40, 120, 4, 20, page_height=40).run_gif([s4], n=3)
    plan.close()


@pytest.mark.gpu
def test_gpu_one_page_is_the_old_entries(vb):
    rng = np.random.default_rng(9)
    for bands in (1, 3, 4):
        a = rng.integers(0, 256, (300, 410, bands), dtype=np.uint8)
        old = vb.Image(a).thumbnail_image(100)
        new = vb.Image(a, page_height=300).thumbnail_image(100)
        assert new.page_height is None and np.array_equal(new.numpy(), old.numpy())
        assert np.array_equal(vb.Image(a, page_height=7).thumbnail_image(100).numpy(), old.numpy())  # 7 does not divide 300
        plan_old = vb.ThumbnailPlan(410, 300, bands, 100)
        plan_new = vb.ThumbnailPlan(410, 300, bands, 100, page_height=300)
        assert plan_old.kernel == plan_new.kernel and plan_new.out_page_height is None
        assert np.array_equal(plan_old.run_host(a[None]), plan_new.run_host(a[None]))
        plan_old.close()
        plan_new.close()
    s = gif_streams()["writer-rgba"]
    assert np.array_equal(vb.thumbnail_buffer(s, 50, page=0, n=1, return_page_height=True)[0], vb.thumbnail_buffer(s, 50))
    w, h, bands, _ = vb.gif_geometry(s)
    plan = vb.ThumbnailPlan(w, h, bands, 50)
    assert np.array_equal(plan.run_gif([s], page=0, n=1), plan.run_gif([s]))
    plan.close()

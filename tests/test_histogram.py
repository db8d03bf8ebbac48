"""vips_hist_find, vips_hist_equal and vips_hist_local on the device (histogram.cu).

CPU: the reference's own hist_find.c / statistic.c, hist_cum.c, hist_norm.c and hist_local.c under oracle/_ref
(ref_hist_*.c) against numpy's counts; hist_equal's LUT from the host compile of the device's per-entry arithmetic
(vb200_debug_hist_equal_lut_host) against the reference chain find -> cum -> norm -> cast; hist_local's staging, window
update and element arithmetic compiled for the host (vb200_debug_hist_local_host), staged and unstaged, against
hist_local.c; the refusals that need no device.  The reference's answers are recorded in
tests/golden/hist_ref_results.json.gz for machines whose oracle/_ref lacks the histogram entry points (see below).
GPU: every op against the oracle and the host twin, at tile seams, past 65 535 rows and columns, from device images at
padded pitches and off-grid bases into host, device and caller buffers, in chains, and the 2^32-pixel refusal."""
import atexit
import ctypes as C
import gzip
import json
import os

import numpy as np
import pytest

from oracle import pyref

UCHAR, USHORT, UINT = 0, 2, 4
DT = {UCHAR: np.uint8, USHORT: np.uint16, UINT: np.uint32}


# ------------------------------------------------------------------------------------------------ the reference
#
# The reference's answers come from oracle/_ref/libvipsref.so when it carries the ref_hist_* entry points (built from the
# reference's sources by oracle/ref_shim/ref_hist_*.c).  Elsewhere -- no reference sources, or a library built before
# those entry points existed -- they come from tests/golden/hist_ref_results.json.gz, written by a run of this file with
# the library present and VB200_REF_RECORD=1, in the form oracle/pyref.py records its own answers: an array as its
# shape, dtype and a digest of its values (pyref.Recorded, which np.array_equal compares by that digest).

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hist_ref_results.json.gz")
_REF = None
_RECORDED = None
_NEW = {}


def ref():
    """the reference library with the histogram entry points, or None"""
    global _REF
    if _REF is None:
        _REF = False
        if pyref.live():
            L = C.CDLL(pyref.PATH)
            if hasattr(L, "ref_hist_find") and hasattr(L, "ref_hist_equal_lut") and hasattr(L, "ref_hist_local"):
                L.ref_image_new_from_memory.restype = C.c_void_p
                L.ref_image_new_from_memory.argtypes = [C.c_void_p] + [C.c_int] * 5
                for f in ("ref_image_width", "ref_image_height", "ref_image_bands", "ref_image_format"):
                    getattr(L, f).argtypes = [C.c_void_p]
                L.ref_image_write_to_memory.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
                L.ref_error.restype = C.c_char_p
                L.ref_hist_find.restype = C.c_void_p
                L.ref_hist_find.argtypes = [C.c_void_p, C.c_int]
                L.ref_hist_equal_lut.restype = C.c_void_p
                L.ref_hist_equal_lut.argtypes = [C.c_void_p, C.c_int]
                L.ref_hist_local.restype = C.c_void_p
                L.ref_hist_local.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
                _REF = L
    return _REF or None


def _save_new():
    old = {}
    if os.path.exists(GOLDEN):
        with gzip.open(GOLDEN, "rt") as f:
            old = json.load(f)
    old.update(_NEW)
    with gzip.GzipFile(GOLDEN, "wb", mtime=0) as f:
        f.write(json.dumps(old, sort_keys=True, separators=(",", ":")).encode())


def _answer(name, args, compute):
    """the reference's answer to name(*args): computed by the library when it is here, else the recorded one"""
    global _RECORDED
    key = pyref._key("hist", name, args)
    if ref() is not None:
        v = compute()
        if os.environ.get("VB200_REF_RECORD"):
            if not _NEW:
                atexit.register(_save_new)
            _NEW[key] = {"error": v} if isinstance(v, str) else pyref._encode(v)
        return v
    if _RECORDED is None:
        with gzip.open(GOLDEN, "rt") as f:
            _RECORDED = json.load(f)
    if key not in _RECORDED:
        raise KeyError("no recorded reference answer for %s%r; record it with oracle/_ref built and VB200_REF_RECORD=1" % (name, args))
    e = _RECORDED[key]
    return e["error"] if isinstance(e, dict) else pyref._decode(e)


def _run(fn, a, *args):
    """a (h, w, bands) array through a ref_* entry -> (array, format), or the reference's error text"""
    L = ref()
    a = np.ascontiguousarray(a)
    fmt = {np.dtype(np.uint8): UCHAR, np.dtype(np.uint16): USHORT}[a.dtype]
    im = L.ref_image_new_from_memory(a.ctypes.data, a.shape[1], a.shape[0], a.shape[2], fmt, 1 if a.shape[2] < 3 else 22)
    out = getattr(L, fn)(im, *args)
    if not out:
        return L.ref_error().decode()
    w, h, b, f = L.ref_image_width(out), L.ref_image_height(out), L.ref_image_bands(out), L.ref_image_format(out)
    res = np.empty((h, w, b), DT[f])
    assert L.ref_image_write_to_memory(out, res.ctypes.data, 0, 0) == 0
    return res, f


def _ref_call(fn, a, *args, keep=lambda v: v):
    """keep: the part of the answer the tests use, recorded as such"""
    def compute():
        v = _run(fn, a, *args)
        return v if isinstance(v, str) else keep(v)
    v = _answer(fn, (a,) + args, compute)
    if isinstance(v, str):
        raise RuntimeError(v)
    return v


def ref_hist_find(a, band=-1):
    """(the histogram as a (1, width, bands) array, its format)"""
    return _ref_call("ref_hist_find", a, band)


def ref_hist_equal_lut(a, band=-1):
    """hist_equal's LUT as a (width, bands) array"""
    return _ref_call("ref_hist_equal_lut", a, band, keep=lambda v: v[0][0])


def ref_hist_local(a, w, h, max_slope):
    return _ref_call("ref_hist_local", a, w, h, max_slope, keep=lambda v: v[0])


def numpy_hist(a, band=-1):
    """hist_find.c's rules restated: uchar band -1 256 wide, else as wide as the largest value seen plus one"""
    sel = a if band < 0 else a[:, :, band:band + 1]
    width = 256 if (a.dtype == np.uint8 and band < 0) else int(sel.max()) + 1
    return np.stack([np.bincount(sel[:, :, b].ravel(), minlength=width)[:width] for b in range(sel.shape[2])], 1).astype(np.uint32)


def apply_lut(a, lut):
    """maplut.c: index clipped to the last entry; a one-band table maps every band"""
    idx = np.minimum(a.astype(np.int64), lut.shape[0] - 1)
    if lut.shape[1] == 1:
        return lut[:, 0][idx]
    return np.stack([lut[:, b][idx[:, :, b]] for b in range(a.shape[2])], 2)


# ------------------------------------------------------------------------------------------------ inputs

def hist_images():
    """(name, array): uchar / ushort, 1-4 bands, narrow ranges, constants, 1 x 1 and 1 x N"""
    rng = np.random.default_rng(7)
    out = []
    for dt, top in ((np.uint8, 256), (np.uint16, 65536)):
        for bands in (1, 2, 3, 4):
            out.append(("%s full %d" % (np.dtype(dt).name, bands), rng.integers(0, top, (23, 31, bands)).astype(dt)))
            out.append(("%s narrow %d" % (np.dtype(dt).name, bands), rng.integers(0, 40 if dt == np.uint8 else 700, (19, 13, bands)).astype(dt)))
        out.append(("%s constant" % np.dtype(dt).name, np.full((9, 11, 3), 5, dt)))
        out.append(("%s zero" % np.dtype(dt).name, np.zeros((4, 6, 1), dt)))
        out.append(("%s 1x1" % np.dtype(dt).name, np.full((1, 1, 2), 3, dt)))
        out.append(("%s 1xN" % np.dtype(dt).name, rng.integers(0, 90, (1, 57, 3)).astype(dt)))
        out.append(("%s Nx1" % np.dtype(dt).name, rng.integers(0, 90, (57, 1, 1)).astype(dt)))
        # bands with very different ranges: a band's LUT narrower than another band's values (maplut clipping)
        a = rng.integers(0, 30, (21, 17, 3)).astype(dt)
        a[:, :, 1] = rng.integers(0, 200, (21, 17)).astype(dt)
        out.append(("%s mixed ranges" % np.dtype(dt).name, a))
    return out


def local_image(rng, h, w, bands):
    a = rng.integers(0, 256, (h, w, bands)).astype(np.uint8)
    a[rng.random((h, w, bands)) < 0.3] = 128  # peaks above max_slope
    return a


# ------------------------------------------------------------------------------------------------ CPU

def test_reference_hist_find_counts():
    for name, a in hist_images():
        for band in [-1] + list(range(a.shape[2])):
            got, fmt = ref_hist_find(a, band)
            want = numpy_hist(a, band)
            assert fmt == UINT and got.dtype == np.uint32 and tuple(got.shape) == (1,) + want.shape, (name, band)
            assert np.array_equal(got, want[None]), (name, band)


def test_hist_equal_lut_host_twin_matches_reference():
    """the twin's LUT from the histogram (numpy's, which is the reference's: test above) against the reference chain's"""
    import libvips_b200 as vb
    for name, a in hist_images():
        for band in [-1] + list(range(a.shape[2])):
            want = ref_hist_equal_lut(a, band)
            got = vb.hist_equal_lut_host_twin(numpy_hist(a, band), a.dtype)
            assert got.dtype == want.dtype and tuple(got.shape) == tuple(want.shape), (name, band)
            assert np.array_equal(got, want), (name, band, pyref.difference(got, want))


LOCAL_WINDOWS = [(1, 1), (2, 2), (3, 3), (4, 7), (8, 5), (15, 15), (16, 16), (17, 9), (31, 32), (33, 33), (63, 63), (64, 2),
                 (2, 40)]


@pytest.mark.parametrize("bands", [1, 2, 3, 4])
def test_hist_local_host_twin_matches_reference(bands):
    import libvips_b200 as vb
    rng = np.random.default_rng(100 + bands)
    a = local_image(rng, 70, 150, bands)
    for (w, h) in LOCAL_WINDOWS:
        for m in (0, 1, 3, 255):
            want = ref_hist_local(a, w, h, m)
            for staged in (None, False):
                got = vb.hist_local_host_twin(a, w, h, m, staged)
                assert np.array_equal(got, want), (w, h, m, staged, pyref.difference(got, want))


def test_hist_local_host_twin_window_is_image_and_narrow_images():
    import libvips_b200 as vb
    rng = np.random.default_rng(5)
    # window equal to the image, and images narrower than two tiles (mirrored edges meet)
    for (ih, iw, w, h) in ((9, 13, 13, 9), (40, 40, 40, 40), (5, 200, 150, 5), (33, 129, 129, 33), (1, 1, 1, 1), (3, 2, 2, 3)):
        a = local_image(rng, ih, iw, 3)
        for m in (0, 3):
            want = ref_hist_local(a, w, h, m)
            for staged in (None, False, True):
                assert np.array_equal(vb.hist_local_host_twin(a, w, h, m, staged), want), (ih, iw, w, h, m, staged)


def test_reference_refuses_large_window():
    a = np.zeros((10, 12, 1), np.uint8)
    with pytest.raises(RuntimeError, match="window too large"):
        ref_hist_local(a, 13, 3, 0)


def test_host_twin_refusals():
    import libvips_b200 as vb
    a = np.zeros((10, 12, 1), np.uint8)
    with pytest.raises(vb.Error, match="window too large"):
        vb.hist_local_host_twin(a, 13, 3)
    with pytest.raises(vb.Error, match="window too large"):
        vb.hist_local_host_twin(a, 3, 11)
    with pytest.raises(vb.Error, match="overflows int"):
        vb.hist_local_host_twin(np.zeros((3000, 3000, 1), np.uint8), 2897, 2897)


def test_standalone_refusals_before_the_device():
    """refusals that need no image come from the constructor, before any device call"""
    import libvips_b200 as vb
    im = vb.Image(np.zeros((16, 16, 1), np.uint8))
    for (w, h, m, what) in ((2897, 2897, 0, "overflows int"), (8388608, 1, 0, "overflows int"), (0, 3, 0, "window too large"),
                            (3, 3, -1, "max_slope")):
        with pytest.raises(vb.Error, match=what):
            im.hist_local(w, h, m)


# ------------------------------------------------------------------------------------------------ GPU

def _reason(vb, rc):
    assert rc == -1
    msg = vb.lib().vb200_error_buffer().decode(errors="replace")
    vb.lib().vb200_error_clear()
    return msg.strip().split(": ", 1)[1]


@pytest.mark.gpu
def test_device_hist_find_and_equal_match_reference(vb):
    for name, a in hist_images():
        im = vb.Image(a)
        for band in [-1] + list(range(a.shape[2])):
            got = im.hist_find(band)
            want = ref_hist_find(a, band)[0]
            assert got.array.dtype == np.uint32 and got.interpretation == 10, name
            assert got.array.shape == tuple(want.shape) and np.array_equal(got.array, want), (name, band)
            # the device's LUT, seen through maplut, is the reference's (compared by digest where the answer is recorded)
            lut = vb.hist_equal_lut_host_twin(numpy_hist(a, band), a.dtype)
            assert np.array_equal(lut, ref_hist_equal_lut(a, band)), (name, band)
            eq = im.hist_equal(band)
            assert eq.array.dtype == a.dtype and np.array_equal(eq.array, apply_lut(a, lut)), (name, band)


# sizes around the 128 x 16 tile and the 32-lane / 256-thread seams
SEAM_SHAPES = [(15, 127), (16, 128), (17, 129), (31, 255), (33, 257), (48, 383), (65, 130)]


def seam_cases():
    """(image, window width, window height, max_slope): windows cut by every CTA, warp and tile seam, and windows whose
    staged tile does not fit in shared memory (the unstaged path)"""
    rng = np.random.default_rng(9)
    for (h, w) in SEAM_SHAPES:
        for bands in (1, 3, 4):
            a = local_image(rng, h, w, bands)
            for (ww, wh) in ((1, 1), (3, 3), (8, 5), (16, 15), (17, 16), (64, 64), (65, 33)):
                if ww <= w and wh <= h:
                    for m in (0, 3, 255):
                        yield a, ww, wh, m
    a = local_image(rng, 300, 400, 3)
    for (ww, wh) in ((300, 200), (400, 300)):
        yield a, ww, wh, 3


def test_hist_local_host_twin_matches_reference_at_seams():
    import libvips_b200 as vb
    for a, ww, wh, m in seam_cases():
        want = ref_hist_local(a, ww, wh, m)
        assert np.array_equal(vb.hist_local_host_twin(a, ww, wh, m), want), (a.shape, ww, wh, m)


@pytest.mark.gpu
def test_device_hist_local_matches_reference_and_twin(vb):
    for a, ww, wh, m in seam_cases():
        got = vb.Image(a).hist_local(ww, wh, m).array
        want = ref_hist_local(a, ww, wh, m)
        assert np.array_equal(got, want), (a.shape, ww, wh, m, pyref.difference(got, want))
        assert np.array_equal(got, vb.hist_local_host_twin(a, ww, wh, m)), (a.shape, ww, wh, m)
    # every CPU case of the host twin, on the device
    for bands in (1, 2, 3, 4):
        a = local_image(np.random.default_rng(100 + bands), 70, 150, bands)
        for (ww, wh) in LOCAL_WINDOWS:
            for m in (0, 1, 3, 255):
                assert np.array_equal(vb.Image(a).hist_local(ww, wh, m).array, ref_hist_local(a, ww, wh, m)), (bands, ww, wh, m)


@pytest.mark.gpu
def test_device_grid_limits(vb):
    rng = np.random.default_rng(3)
    for shape in ((70000, 17, 3), (17, 70000, 3)):
        a = local_image(rng, *shape)
        im = vb.Image(a)
        assert np.array_equal(im.hist_find().array[0], numpy_hist(a))
        assert np.array_equal(im.hist_find(1).array[0], numpy_hist(a, 1))
        want_lut = vb.hist_equal_lut_host_twin(numpy_hist(a), np.uint8)
        assert np.array_equal(im.hist_equal().array, apply_lut(a, want_lut))
        b = a.astype(np.uint16) * 201
        assert np.array_equal(vb.Image(b).hist_find().array[0], numpy_hist(b))
        for (ww, wh) in ((5, 5), (17, 17)):
            assert np.array_equal(im.hist_local(ww, wh, 3).array, vb.hist_local_host_twin(a, ww, wh, 3)), (shape, ww, wh)


@pytest.mark.gpu
def test_device_resident_inputs_and_outputs(vb):
    """the wants are numpy's histogram, the twin's LUT and the twin's hist_local, each pinned to the reference above"""
    import test_device_images as D
    rng = np.random.default_rng(4)
    L = vb.lib()
    for dt in (np.uint8, np.uint16):
        for bands in (1, 3):
            a = (rng.integers(0, 256, (29, 37, bands)) * (1 if dt == np.uint8 else 97)).astype(dt)
            cases = [("hist_find", lambda i, o: L.vb200_hist_find(i, o, -1), numpy_hist(a)[None]),
                     ("hist_equal", lambda i, o: L.vb200_hist_equal(i, o, 0),
                      apply_lut(a, vb.hist_equal_lut_host_twin(numpy_hist(a, 0), dt)))]
            if dt == np.uint8:
                cases.append(("hist_local", lambda i, o: L.vb200_hist_local(i, o, 9, 7, 3), vb.hist_local_host_twin(a, 9, 7, 3)))
            for layout in D.layouts(dt, bands):
                cin, buf = D.device_image(a, layout, 1)
                for what, call, want in cases:
                    # library-allocated device output
                    cout = vb.CImage()
                    cout.where = vb.DEVICE
                    assert call(C.byref(cin), C.byref(cout)) == 0, (what, layout)
                    got = D.take_device(cout)
                    assert got.dtype == want.dtype and np.array_equal(got, want), (what, layout, dt, bands)
                    # a host input's result lands on the host
                    hin, cout = vb.Image(a)._c(), vb.CImage()
                    assert call(C.byref(hin), C.byref(cout)) == 0 and cout.where == vb.HOST
                    assert np.array_equal(vb.Image._take(cout).array, want), (what, layout)
                    # the caller's device buffer at a padded pitch
                    h, w, b = want.shape
                    line = w * b * want.itemsize
                    obuf = D.Buf(h, line, 0, line + 8 * want.itemsize)
                    cout = vb.CImage(w, h, b, vb.FORMATS[want.dtype], 0, vb.DEVICE, C.c_void_p(obuf.ptr), line + 8 * want.itemsize)
                    assert call(C.byref(cin), C.byref(cout)) == 0, (what, layout)
                    assert np.array_equal(obuf.rows(want.dtype, w, b), want), (what, layout)
                    obuf.assert_outside_untouched(what)
                buf.assert_outside_untouched(layout)


@pytest.mark.gpu
def test_chains_equal_standalone_calls(vb):
    rng = np.random.default_rng(8)
    imgs = [local_image(rng, h, w, 3) for (h, w) in ((120, 160), (97, 203), (64, 64), (150, 90))]
    got = vb.Chain().resize(0.7).hist_local(15, 13, 3).sharpen().run(imgs)
    for a, g in zip(imgs, got):
        want = vb.Image(a).resize(0.7).hist_local(15, 13, 3).sharpen()
        assert g.array.dtype == want.array.dtype and np.array_equal(g.array, want.array)
    got = vb.Chain().hist_equal().colourspace("lab").run(imgs)
    for a, g in zip(imgs, got):
        want = vb.Image(a).hist_equal().colourspace("lab")
        assert np.array_equal(g.array, want.array)
    got = vb.Chain().hist_equal(1).hist_find().run(imgs)
    for a, g in zip(imgs, got):
        assert np.array_equal(g.array, vb.Image(a).hist_equal(1).hist_find().array)


@pytest.mark.gpu
def test_refusals_alike_standalone_and_chain(vb):
    L = vb.lib()
    im = vb.Image(np.zeros((16, 20, 3), np.uint8))
    imf = vb.Image(np.zeros((16, 20, 3), np.float32))
    cases = [
        ("window too large", im, lambda i, o: L.vb200_hist_local(i, o, 21, 3, 0), lambda c: L.vb200_chain_add_hist_local(c, 21, 3, 0)),
        ("window too large", im, lambda i, o: L.vb200_hist_local(i, o, 3, 17, 0), lambda c: L.vb200_chain_add_hist_local(c, 3, 17, 0)),
        ("overflows int", im, lambda i, o: L.vb200_hist_local(i, o, 4096, 4096, 0), lambda c: L.vb200_chain_add_hist_local(c, 4096, 4096, 0)),
        ("bandno must be -1, or less than 3", im, lambda i, o: L.vb200_hist_find(i, o, 3), lambda c: L.vb200_chain_add_hist_find(c, 3)),
        ("bandno must be -1, or less than 3", im, lambda i, o: L.vb200_hist_equal(i, o, -2), lambda c: L.vb200_chain_add_hist_equal(c, -2)),
        ("cast to uchar or ushort first", imf, lambda i, o: L.vb200_hist_find(i, o, -1), lambda c: L.vb200_chain_add_hist_find(c, -1)),
        ("cast to uchar or ushort first", imf, lambda i, o: L.vb200_hist_equal(i, o, -1), lambda c: L.vb200_chain_add_hist_equal(c, -1)),
        ("image must be uchar", imf, lambda i, o: L.vb200_hist_local(i, o, 3, 3, 0), lambda c: L.vb200_chain_add_hist_local(c, 3, 3, 0)),
    ]
    for what, image, call, add in cases:
        cin, cout = image._c(), vb.CImage()
        launches = vb.launch_count()
        alone = _reason(vb, call(C.byref(cin), C.byref(cout)))
        assert what in alone and not cout.data and vb.launch_count() == launches, (what, alone)
        chain = vb.Chain()
        rc = add(chain._p)
        if rc == 0:  # refused by the image: the same reason from the chain's run
            cin, cout = image._c(), vb.CImage()
            rc = L.vb200_chain_run_host(chain._p, C.byref(cin), C.byref(cout), 1)
        assert _reason(vb, rc) == alone, what
        chain.close()


@pytest.mark.gpu
def test_large_hist_find_declined(vb):
    """65 536 x 65 536 pixels: the reference's DOUBLE histogram, not built on the device; refused with its reason"""
    import torch
    t = torch.zeros(65536 * 65536, dtype=torch.uint8, device="cuda")
    cin = vb.CImage(65536, 65536, 1, UCHAR, 1, vb.DEVICE, C.c_void_p(t.data_ptr()), 65536)
    for call in (vb.lib().vb200_hist_find, vb.lib().vb200_hist_equal):
        cout = vb.CImage()
        assert "2^32 or more pixels" in _reason(vb, call(C.byref(cin), C.byref(cout), -1))
    del t
    torch.cuda.empty_cache()

"""The chain pump for unfused graphs (SURVEY 8f rank 2, vb200_chain_*): a list of operations run over a
batch of host images with every intermediate on the device.  Expected pixels: the oracle's operations
applied one after the other (each pinned to the reference by its own test file)."""
import numpy as np
import pytest

from oracle import pyconv, pyoracle as orc

pytestmark = pytest.mark.gpu


def test_chain_matches_oracle_op_by_op(vb):
    rng = np.random.default_rng(90)
    imgs = [rng.integers(0, 256, s, dtype=np.uint8) for s in ((300, 400, 3), (257, 129, 3), (64, 64, 3), (500, 333, 3))]
    chain = vb.Chain().resize(0.4).gaussblur(1.2, 0.2, "integer").sharpen().colourspace("lab")
    got = chain.run(imgs)
    for a, g in zip(imgs, got):
        want = orc.resize(a, 0.4)
        want = pyconv.gaussblur(want, 1.2, 0.2, "integer")
        want = pyconv.sharpen(want, "srgb")
        want = orc.colourspace(want, "lab", "srgb")
        assert g.numpy().shape == want.shape and np.array_equal(g.numpy(), want)
    # the same chain again (streams and pool are reused), and a different batch size
    again = chain.run(imgs[:2])
    assert all(np.array_equal(x.numpy(), y.numpy()) for x, y in zip(again, got))


def test_chain_equals_standalone_calls(vb):
    rng = np.random.default_rng(91)
    a = rng.integers(0, 256, (240, 320, 4), dtype=np.uint8)
    mask = np.array([[1.0, 2.0, 1.0], [2.0, 4.0, 2.0], [1.0, 2.0, 1.0]])
    got = vb.Chain().premultiply(uchar=True).reduce(2.5, 1.7).unpremultiply(uchar=True).conv(mask, 16.0, 0.0, "integer").run([a])[0]
    step = vb.Image(a).premultiply(uchar=True).reduce(2.5, 1.7).unpremultiply(uchar=True).conv(mask, 16.0, 0.0, "integer")
    assert np.array_equal(got.numpy(), step.numpy())
    # float convsep with a column mask in a chain
    col = np.array([[1.0], [3.0], [5.0], [2.0]])
    got = vb.Chain().convsep(col, 11.0, 1.0, "float").run([a])[0]
    assert np.array_equal(got.numpy(), pyconv.convsep(a, col, 11.0, 1.0, "float"))


def test_chain_errors_surface(vb):
    a = np.zeros((32, 32, 3), np.uint8)
    with pytest.raises(vb.Error, match="reduce factor should be >= 1.0"):
        vb.Chain().reduce(0.5, 2.0).run([a])
    with pytest.raises(vb.Error):
        vb.Chain().colourspace("cmyk").run([a])


# ------------------------------------------------------------------ every chain op against its stand-alone call
U8, I16, F32 = np.uint8, np.int16, np.float32
M33 = np.array([[0.25, -0.5, 0.125], [1.0, 0.75, -0.25], [0.0, 0.5, 0.375]])
MI33 = np.array([[1.0, -2.0, 3.0], [2.0, 5.0, -1.0], [0.0, 4.0, 1.0]])
SEP5 = np.array([[1.0, 4.0, 6.0, 4.0, 1.0]])
CROSS = np.array([[128.0, 255.0, 128.0], [255.0, 255.0, 0.0], [128.0, 255.0, 128.0]])


def _pixels(rng, dt, shape, space=None):
    """the whole range of an integer format, floats in [-20, 280); Lab and LabS inputs in their own ranges"""
    dt = np.dtype(dt)
    if space == "lab":
        a = rng.random(shape).astype(dt)
        a[..., 0] *= 100
        a[..., 1:3] = a[..., 1:3] * 256 - 128
        return a
    if dt.kind == "f":
        return (rng.random(shape) * 300 - 20).astype(dt)
    i = np.iinfo(dt)
    a = rng.integers(i.min, int(i.max) + 1, shape, dtype=np.int64).astype(dt)
    if space == "labs":
        a[..., 0] = np.abs(a[..., 0])
    return a


# (name, formats, band counts, input interpretation (None: B_W below 3 bands, else sRGB), the step on a Chain or an Image):
# the formats and band counts test_device_images.py's OPS table runs each op with, restricted to uchar, short and float
STEPS = [
    ("resize_down", (U8, I16, F32), (3, 4), None, lambda t: t.resize(0.6, 0.0, gap=-1.0)),
    ("resize_up", (U8, I16, F32), (3, 4), None, lambda t: t.resize(1.7, 1.3)),
    ("reduce", (U8, I16, F32), (3, 4), None, lambda t: t.reduce(2.3, 1.7)),
    ("colourspace_srgb_lab", (U8,), (3, 4), "srgb", lambda t: t.colourspace("lab")),
    ("colourspace_labs_lab", (I16,), (3,), "labs", lambda t: t.colourspace("lab")),
    ("colourspace_lab_srgb", (F32,), (3,), "lab", lambda t: t.colourspace("srgb")),
    ("colourspace_bw_srgb", (U8,), (1,), "b-w", lambda t: t.colourspace("srgb")),
    ("conv", (U8, I16, F32), (3, 4), None, lambda t: t.conv(M33, 1.3, 0.5, "float")),
    ("conv_integer", (U8, I16, F32), (3, 4), None, lambda t: t.conv(MI33, 7.0, 1.0, "integer")),
    ("convsep", (U8, I16, F32), (3, 4), None, lambda t: t.convsep(SEP5, 16.0, 0.0, "integer")),
    ("gaussblur", (U8, I16, F32), (3, 4), None, lambda t: t.gaussblur(1.0, 0.2, "float")),
    ("gaussblur_default_ampl", (U8, I16, F32), (3, 4), None, lambda t: t.gaussblur(1.0, 0.0, "integer")),
    ("sharpen", (U8,), (3, 4), None, lambda t: t.sharpen()),
    ("premultiply", (U8, I16, F32), (3, 4), None, lambda t: t.premultiply(255.0)),
    ("unpremultiply", (U8, I16, F32), (3, 4), None, lambda t: t.unpremultiply(255.0)),
    ("premultiply_uchar", (U8,), (2, 3, 4), None, lambda t: t.premultiply(255.0, uchar=True)),
    ("unpremultiply_uchar", (U8,), (2, 3, 4), None, lambda t: t.unpremultiply(255.0, uchar=True)),
    ("morph", (U8,), (1, 3, 4), None, lambda t: t.morph(CROSS, "dilate")),
    ("rank", (U8, I16, F32), (3, 4), None, lambda t: t.rank(3, 3, 2)),
    ("flatten", (U8, I16, F32), (4,), None, lambda t: t.flatten((10.7, 200.2, 33.0))),
]


def _standalone(vb, step, images):
    """the stand-alone call on each image, and the kernel launches each one took"""
    got, launches = [], []
    for im in images:
        before = vb.launch_count()
        got.append(step(im))
        launches.append(vb.launch_count() - before)
    return got, launches


def _chained(vb, chain, images):
    """the chain over each image alone (its launches per image), then over the whole batch"""
    launches = []
    for im in images:
        before = vb.launch_count()
        chain.run([im])
        launches.append(vb.launch_count() - before)
    before = vb.launch_count()
    got = chain.run(images)
    assert vb.launch_count() - before == sum(launches)
    return got, launches


def _same(got, want):
    for g, w in zip(got, want):
        assert g.numpy().dtype == w.numpy().dtype and g.numpy().shape == w.numpy().shape
        assert g.interpretation == w.interpretation
        assert np.array_equal(g.numpy(), w.numpy(), equal_nan=g.numpy().dtype.kind == "f")


@pytest.mark.parametrize("name", [s[0] for s in STEPS])
def test_chain_step_equals_standalone_call(vb, name):
    """each chain op is the stand-alone op's own record: same pixels, format, interpretation and launches, over a batch of
    two images of different sizes"""
    _, formats, bands, space, step = next(s for s in STEPS if s[0] == name)
    rng = np.random.default_rng(92)
    for dt in formats:
        for b in bands:
            images = [vb.Image(_pixels(rng, dt, (h, w, b), space), space) for h, w in ((67, 91), (38, 45))]
            want, want_launches = _standalone(vb, step, images)
            got, launches = _chained(vb, step(vb.Chain()), images)
            _same(got, want)
            assert launches == want_launches, (name, dt, b)


def test_chain_pass_through_steps(vb):
    """steps that hand their input on (gaussblur below sigma 0.2, premultiply of one band) first, inside and last in a
    chain: the stand-alone sequence's pixels and launches"""
    rng = np.random.default_rng(93)
    cases = [
        (1, lambda t: t.gaussblur(0.1).premultiply().resize(0.7).gaussblur(0.1).premultiply().conv(M33).premultiply()),
        (3, lambda t: t.gaussblur(0.1).sharpen().gaussblur(0.1).reduce(1.5, 1.5).gaussblur(0.1)),
    ]
    for b, steps in cases:
        images = [vb.Image(rng.integers(0, 256, (h, w, b), dtype=np.uint8)) for h, w in ((70, 52), (33, 81))]
        want, want_launches = _standalone(vb, steps, images)
        got, launches = _chained(vb, steps(vb.Chain()), images)
        _same(got, want)
        assert launches == want_launches


def _reason(vb, rc):
    """-1, and the error text without its domain"""
    assert rc == -1
    msg = vb.lib().vb200_error_buffer().decode(errors="replace")
    vb.lib().vb200_error_clear()
    return msg.strip().split(": ", 1)[1]


def test_chain_and_standalone_refuse_alike(vb):
    """every refusal that needs no image (no mask, a mask dimension <= 0, a convsep mask that is not 1xn or nx1, a reduce
    factor below 1): the same reason from the stand-alone call and from the chain's add, and *out untouched"""
    import ctypes as C
    L = vb.lib()
    coeff = np.ones(9, np.float64)
    ptr = coeff.ctypes.data_as(C.POINTER(C.c_double))
    masks = {"no mask": None, "zero width": vb.CMask(0, 3, ptr, 1.0, 0.0), "negative height": vb.CMask(3, -1, ptr, 1.0, 0.0),
             "null coefficients": vb.CMask(3, 3, None, 1.0, 0.0)}
    cases = []
    for what, m in masks.items():
        arg = C.byref(m) if m is not None else None
        cases.append((what + " conv", lambda i, o, a=arg: L.vb200_conv(i, o, a, 0), lambda c, a=arg: L.vb200_chain_add_conv(c, a, 0)))
        cases.append((what + " convsep", lambda i, o, a=arg: L.vb200_convsep(i, o, a, 0),
                      lambda c, a=arg: L.vb200_chain_add_convsep(c, a, 0)))
        cases.append((what + " morph", lambda i, o, a=arg: L.vb200_morph(i, o, a, 0), lambda c, a=arg: L.vb200_chain_add_morph(c, a, 0)))
    square = vb.CMask(3, 3, ptr, 1.0, 0.0)
    cases.append(("square convsep", lambda i, o: L.vb200_convsep(i, o, C.byref(square), 0),
                  lambda c: L.vb200_chain_add_convsep(c, C.byref(square), 0)))
    for hs, vs in ((0.5, 2.0), (2.0, 0.5)):
        cases.append(("reduce %g %g" % (hs, vs), lambda i, o, hs=hs, vs=vs: L.vb200_reduce(i, o, hs, vs, 2, 0.0),
                      lambda c, hs=hs, vs=vs: L.vb200_chain_add_reduce(c, hs, vs, 2, 0.0)))
    im = vb.Image(np.zeros((16, 16, 3), np.uint8))
    for what, call, add in cases:
        cin, cout = im._c(), vb.CImage()
        alone = _reason(vb, call(C.byref(cin), C.byref(cout)))
        assert not cout.data and cout.Xsize == 0, what
        chain = vb.Chain()
        assert _reason(vb, add(chain._p)) == alone, what
        chain.close()

"""Every convolution kernel at every mask length.

dev_conv (libvips_b200/csrc/conv.cu) sends a float-precision mask to one of four kernels: convf_dense_kernel (1-D, every
position a tap, 8..64 taps), convf_block_kernel (other 1-D masks of at most 64 positions), convf_line_kernel (1-D masks
with at most 64 non-zero taps) and convf_kernel (everything else); integer precision goes to convi_kernel,
convi_float_kernel or, in vector mode, convi_vector_u8_kernel.  vips_sharpen on 8-bit sRGB is sharpen_fused_kernel up to
15 taps and the unfused chain (colourspace, two convi passes, sharpen_kernel) beyond.  Each kernel has its own schedule
(head / full groups / remainder / tail, sliding coefficient windows, interior and clamped edges), so a slip in one shows
only at some mask lengths and image sizes.  These tests run every length 1..66 plus 80, 127 and 129, as rows and
columns, on images smaller than the mask and larger than a register block, in every format.

Two expectations:
  * the oracle (oracle.pyconv), bit for bit -- itself pinned here to the reference's own convf.c / convi.c / convsep.c /
    sharpen.c at the same kinds of shapes;
  * for float precision, a plain float64 convolution written below (edge-replicating padding, zero taps skipped), within
    one float32 ulp plus 2^-40 of the sum of |term|.  It shares no code with the oracle, so it catches a mistake the
    oracle and a kernel could share: orientation, the centre of even masks, edge handling.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import pyconv, pyref
from oracle import pyoracle as orc

needs_ref = pytest.mark.skipif(not pyref.available(), reason="oracle/_ref not built")

FORMATS = [np.uint8, np.int8, np.uint16, np.int16, np.uint32, np.int32, np.float32]
BANDS = (1, 3, 4)
LENGTHS = list(range(1, 67)) + [80, 127, 129]
FAMILIES = ("gauss", "rand", "head0", "tail0", "sparse", "spread", "zero", "first", "last")
RB = 8  # outputs per thread of convf_block_kernel / convf_dense_kernel
# dev_conv's environment switches, in the order the kernels are tried
ENVS = {"default": None, "no_dense": "VB200_NO_CONV_DENSE", "no_block": "VB200_NO_CONV_BLOCK"}
# sharpen: gaussmat(sigma, 0.1) integer tap counts 1, 3, ..., 15 (sharpen_fused_kernel) and 17, 21 (unfused)
SHARPEN_SIGMAS = {0.3: 1, 0.5: 3, 1.0: 5, 1.5: 7, 1.9: 9, 2.4: 11, 3.0: 13, 3.5: 15}
WIDE_SHARPEN_SIGMAS = {4.0: 17, 5.0: 21}
LUTS = ({"x1": 2.0, "m1": 0.0, "m2": 3.0, "y2": 10.0, "y3": 20.0}, {"x1": 1.0, "m1": 0.5, "m2": 5.0, "y2": 20.0, "y3": 5.0})


# ------------------------------------------------------------------------------------------------ helpers

def image(rng, dt, shape, special=False):
    """random pixels over the whole range of an integer format; for float, [-75, 225) and, with special, NaN and +-Inf"""
    dt = np.dtype(dt)
    if dt.kind == "f":
        a = ((rng.random(shape) - 0.25) * 300).astype(dt)
        if special and a.size >= 3:
            a.reshape(-1)[rng.choice(a.size, 3, replace=False)] = [np.nan, np.inf, -np.inf]
        return a
    i = np.iinfo(dt)
    return rng.integers(i.min, int(i.max) + 1, shape, dtype=np.int64).astype(dt)


def photo(rng, h, w, b):
    """smooth content with texture (as in test_pipeline.py): small L differences reach the LUT's centre and both slopes"""
    y, x = np.mgrid[0:h, 0:w]
    base = 128 + 90 * np.sin(x / 17.0) * np.cos(y / 23.0)
    out = np.clip(base[:, :, None] + rng.normal(0, 6, (h, w, b)) + np.array([10, -20, 30, 0][:b]), 0, 255).astype(np.uint8)
    if b == 4:
        out[:, :, 3] = rng.integers(0, 256, (h, w), dtype=np.uint8)
    return out


def same(got, want, what=""):
    """bit-exact, NaN equal to NaN"""
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    bad = got != want
    if got.dtype.kind == "f":
        bad &= ~(np.isnan(got) & np.isnan(want))
    assert not bad.any(), (what, np.argwhere(bad)[:5], got[bad][:5], want[bad][:5])


def ref64(a, mask, scale=1.0, offset=0.0):
    """vips_conv at float precision in float64: VIPS_EXTEND_COPY padding of (n // 2, n - 1 - n // 2) per axis, taps
    mask / scale in row-major order with zero taps skipped (an all-zero mask keeps position 0), offset + sum of c * v.
    Returns the sum and the sum of |c * v| (the scale of its rounding error)."""
    m = np.atleast_2d(np.asarray(mask, np.float64))
    mh, mw = m.shape
    c = (m / scale).ravel()
    taps = [(i, c[i]) for i in np.flatnonzero(c)] or [(0, 0.0)]
    a = a if a.ndim == 3 else a[:, :, None]
    h, w = a.shape[:2]
    p = np.pad(a.astype(np.float64), ((mh // 2, mh - 1 - mh // 2), (mw // 2, mw - 1 - mw // 2), (0, 0)), mode="edge")
    s = np.full(a.shape, float(offset))
    mag = np.zeros(a.shape)
    with np.errstate(invalid="ignore", over="ignore"):
        for i, ci in taps:
            y, x = divmod(int(i), mw)
            t = ci * p[y:y + h, x:x + w]
            s += t
            mag += np.abs(t)
    return s, mag


def ref64_sep(a, mask, scale=1.0, offset=0.0):
    """vips_convsep at float precision: conv(M) with the offset, rounded to float as convf stores it, then conv(rot90(M))
    with offset 0 -- a 1 x n row is followed by the same taps as a column, an n x 1 column by its taps reversed as a row"""
    m = np.atleast_2d(np.asarray(mask, np.float64))
    second = m.reshape(-1, 1) if m.shape[0] == 1 else m.ravel()[::-1].reshape(1, -1)
    mid, _ = ref64(a, m, scale, offset)
    with np.errstate(over="ignore"):
        return ref64(mid.astype(np.float32), second, scale, 0.0)


def within(got, want, mag, what=""):
    """|got - want| <= ulp32(want) + 2^-40 * sum |c * v|; NaN where want is NaN, the same infinity where it is infinite"""
    assert got.shape == want.shape, (what, got.shape, want.shape)
    g = got.astype(np.float64)
    nan, inf = np.isnan(want), np.isinf(want)
    assert np.array_equal(np.isnan(g), nan), (what, "NaN pattern")
    assert np.array_equal(g[inf], want[inf]), (what, "infinities")
    fin = ~(nan | inf)
    err = np.abs(g[fin] - want[fin])
    tol = np.spacing(np.abs(want[fin]).astype(np.float32)).astype(np.float64) + 2.0 ** -40 * mag[fin]
    if err.size:
        k = np.argmax(err - tol)
        assert err[k] <= tol[k], (what, "error %g > %g at value %r" % (err[k], tol[k], want[fin][k]))


def line_mask(n, family, seed):
    """a 1-D mask of n taps, (coefficients, scale, offset)"""
    rng = np.random.default_rng(seed)
    if family == "gauss":  # dense, positive, centred between taps for even n
        x = np.arange(n) - (n - 1) / 2
        m = np.exp(-x * x / (2 * (n / 4 + 0.5) ** 2))
        return m, float(m.sum()), 0.0
    m = rng.uniform(0.1, 1.0, n) * rng.choice([-1.0, 1.0], n)  # dense, mixed signs, no symmetry
    k = min(8, n)
    if family == "head0":  # zero taps in the first window, position 0 among them
        m[0] = 0
        m[1:k][rng.random(k - 1) < 0.35] = 0
    elif family == "tail0":  # zero taps in the last window, position n - 1 among them
        m[n - 1] = 0
        m[n - k:n - 1][rng.random(k - 1) < 0.35] = 0
    elif family == "sparse":  # ~20 % zeros anywhere, both end taps kept
        m[1:-1][rng.random(max(0, n - 2)) < 0.2] = 0
    elif family == "spread":  # at most 64 taps spread over the whole length, both ends included
        keep = np.unique(np.linspace(0, n - 1, min(n, 64)).round().astype(int))
        m[np.setdiff1d(np.arange(n), keep)] = 0
    elif family == "zero":
        m[:] = 0
    elif family == "first":
        m[:] = 0
        m[0] = 1.75
    elif family == "last":
        m[:] = 0
        m[n - 1] = -0.625
    return m, 3.25, -1.5


def oriented(m, orient):
    return m[None, :] if orient == "row" else m[:, None]


def expected_kernel(mask, scale, env="default"):
    """the kernel dev_conv picks for a float-precision mask (conv.cu, the dense_ok / block_ok / line_h / line_v
    predicates): dense / block / line with _h or _v, or convf"""
    m = np.atleast_2d(np.asarray(mask, np.float64))
    mh, mw = m.shape
    c = m.ravel() / scale
    nnz = max(1, np.count_nonzero(c))  # the all-zero mask keeps one tap
    line_h, line_v = mh == 1 and nnz <= 64, mw == 1 and nnz <= 64
    block = (line_h or line_v) and c.size <= 64 and env != "no_block" and np.count_nonzero(c) > 0
    dense = block and c.size >= RB and np.count_nonzero(c) == c.size and env != "no_dense"
    side = "_h" if line_h else "_v"
    if dense:
        return "dense" + side
    if block:
        return "block" + side
    if line_h or line_v:
        return "line" + side
    return "convf"


def env_kernels(mask, scale):
    """{kernel: env} for the environments that reach distinct kernels, in ENVS order"""
    out = {}
    for env in ENVS:
        out.setdefault(expected_kernel(mask, scale, env), env)
    return out


def set_env(monkeypatch, env):
    for var in ENVS.values():
        if var:
            monkeypatch.delenv(var, raising=False)
    if ENVS[env]:
        monkeypatch.setenv(ENVS[env], "1")


def line_images(n, orient, seed):
    """(array) for one mask: 1 x 1, one row / column, 7 x 9 and 9 x 7, narrower than half the mask along its axis, long
    along its axis (the interior path), and a ragged 61 x 83; formats and bands rotate with n so every kernel sees all"""
    rng = np.random.default_rng(seed)
    k = max(1, (n - 1) // 2)
    along = (5, k) if orient == "row" else (k, 5)
    long = (3, 2 * n + 40) if orient == "row" else (2 * n + 40, 3)
    out = []
    for i, (h, w) in enumerate([(1, 1), (1, 37), (37, 1), (7, 9), (9, 7), along, long, (61, 83)]):
        dt = FORMATS[(seed + i) % len(FORMATS)]
        b = BANDS[(seed // 7 + i) % len(BANDS)]
        out.append(image(rng, dt, (h, w, b), special=(h, w) in ((7, 9), (61, 83))))
    return out


def line_cases():
    for n in LENGTHS:
        for orient in ("row", "col"):
            seen = []
            for fi, family in enumerate(FAMILIES):
                seed = n * 100 + fi * 10 + (orient == "col")
                m, scale, offset = line_mask(n, family, seed)
                if family == "spread" and n <= 64 or any(np.array_equal(m, s) for s in seen):
                    continue  # the same mask as an earlier family
                seen.append(m)
                mask = oriented(m, orient)
                kern = "/".join(env_kernels(mask, scale))
                yield pytest.param(n, orient, family, seed, id="n%d-%s-%s-%s" % (n, orient, family, kern))


# ------------------------------------------------------------------------------------------------ CPU

def test_expected_kernel_covers_every_kernel():
    seen = set()
    for p in line_cases():
        n, orient, family, seed = p.values
        m, scale, _ = line_mask(n, family, seed)
        seen.update(env_kernels(oriented(m, orient), scale))
    assert seen == {"dense_h", "dense_v", "block_h", "block_v", "line_h", "line_v", "convf"}
    # the boundaries of conv.cu's predicates
    assert expected_kernel(np.ones((1, 8)), 1) == "dense_h" and expected_kernel(np.ones((1, 7)), 1) == "block_h"
    assert expected_kernel(np.ones((64, 1)), 1) == "dense_v" and expected_kernel(np.ones((65, 1)), 1) == "convf"
    assert expected_kernel(np.ones((1, 64)), 1, "no_dense") == "block_h"
    assert expected_kernel(np.ones((1, 64)), 1, "no_block") == "line_h"
    assert expected_kernel(np.zeros((1, 9)), 1) == "line_h"
    assert expected_kernel(np.ones((3, 3)), 1) == "convf"


@pytest.mark.parametrize("n", [1, 2, 8, 16, 17, 33, 64, 65, 100])
@pytest.mark.parametrize("orient", ["row", "col"])
def test_float64_reference_matches_oracle(n, orient):
    """the float64 reference and the oracle agree within the tolerance the GPU tests use (conv and convsep)"""
    rng = np.random.default_rng(n * 2 + (orient == "col"))
    m = rng.uniform(-1, 1, n)
    m[rng.random(n) < 0.2] = 0
    mask = oriented(m, orient)
    for dt in (np.uint8, np.int32, np.float32):
        for shape in ((1, 1, 1), (9, 2, 3), (2, 9, 1), (23, 31, 3)):
            a = image(rng, dt, shape, special=True)
            within(pyconv.conv(a, mask, 1.7, -0.5, "float"), *ref64(a, mask, 1.7, -0.5), what=(dt, shape, "conv"))
            within(pyconv.convsep(a, mask, 1.7, -0.5, "float"), *ref64_sep(a, mask, 1.7, -0.5), what=(dt, shape, "convsep"))


def test_float64_reference_is_not_the_transposed_or_reflected_convolution():
    """the reference pins orientation and the centre of an even mask: a reflected mask, or a centre one tap off (for an
    even mask, position (n - 1) // 2 instead of n // 2), fails"""
    rng = np.random.default_rng(3)
    a = image(rng, np.float32, (11, 13, 1))
    for m in (np.array([[1.0, 4.0, -2.0, 0.5]]), np.array([[1.0, 4.0, -2.0, 0.5, 3.0]])):
        got = pyconv.conv(a, m, 1.0, 0.0, "float")
        within(got, *ref64(a, m))
        with pytest.raises(AssertionError):
            within(got, *ref64(a, m[:, ::-1]))
        # a leading zero tap moves the centre one position right of the original taps, a trailing one (odd n) left
        off = np.concatenate([[[0.0]], m], axis=1) if m.shape[1] % 2 == 0 else np.concatenate([m, [[0.0]]], axis=1)
        with pytest.raises(AssertionError):
            within(got, *ref64(a, off))
        with pytest.raises(AssertionError):
            within(pyconv.conv(a, m.T.copy(), 1.0, 0.0, "float"), *ref64(a, m))


PIN_LENGTHS = [1, 2, 3, 4, 8, 9, 15, 16, 17, 24, 33, 64, 65, 100]
PIN_SHAPES = [(1, 1), (2, 9), (9, 2), (13, 17)]


def pin_mask(n, seed, precision):
    """asymmetric, zero end taps where there is room, negative and fractional scale / offset"""
    rng = np.random.default_rng(seed)
    m = rng.uniform(-1, 1, n)
    if n > 2:
        m[0] = m[-1] = 0
    if precision == "integer":
        return np.rint(m * 20), (-2.6 if seed % 2 else 13.5), (-3.5 if seed % 2 else 2.5)
    return m, (-1.3 if seed % 2 else 0.37), (-2.25 if seed % 2 else 0.5)


@needs_ref
@pytest.mark.parametrize("n", PIN_LENGTHS)
@pytest.mark.parametrize("orient", ["row", "col"])
@pytest.mark.parametrize("precision", ["float", "integer"])
def test_oracle_conv_matches_reference_at_every_length(n, orient, precision):
    """the oracle's conv and convsep against the reference's own convf.c / convi.c / convsep.c / rot.c"""
    seed = n * 4 + (orient == "col") * 2 + (precision == "integer")
    m, scale, offset = pin_mask(n, seed, precision)
    mask = oriented(m, orient)
    rng = np.random.default_rng(seed)
    for i, (h, w) in enumerate(PIN_SHAPES):
        a = image(rng, FORMATS[(seed + i) % len(FORMATS)], (h, w, BANDS[i % 3]))
        what = (a.shape, a.dtype)
        got, want = pyconv.conv(a, mask, scale, offset, precision), pyconv.ref_conv(a, mask, scale, offset, precision)
        assert np.array_equal(got, want, equal_nan=True), ("conv",) + what
        got, want = pyconv.convsep(a, mask, scale, offset, precision), pyconv.ref_convsep(a, mask, scale, offset, precision)
        assert np.array_equal(got, want, equal_nan=True), ("convsep",) + what


@needs_ref
@pytest.mark.parametrize("sigma", [0.3, 0.5, 1.0, 1.5, 1.9, 2.4, 3.0, 3.5, 4.0, 5.0, 8.0])
def test_oracle_sharpen_matches_reference_at_every_length(sigma):
    """vips_sharpen from 1 to 35 taps against the reference's sharpen.c, on images smaller than the mask"""
    rng = np.random.default_rng(int(sigma * 10))
    kw = LUTS[int(sigma * 10) % 2]
    for shape in ((1, 1, 3), (2, 33, 3), (33, 2, 3), (40, 70, 3)):
        for a in (image(rng, np.uint8, shape), np.full(shape, 255, np.uint8), np.zeros(shape, np.uint8)):
            assert np.array_equal(pyconv.sharpen(a, "srgb", sigma=sigma, **kw), pyconv.ref_sharpen(a, "srgb", sigma=sigma, **kw)), shape


def test_sharpen_tap_counts():
    """the sigmas the sharpen tests use give the tap counts they are named for"""
    for sigma, n in {**SHARPEN_SIGMAS, **WIDE_SHARPEN_SIGMAS}.items():
        assert pyconv.gaussmat(sigma, 0.1, True, "integer")[0].shape == (1, n), sigma
    for sigma, n in {4.5: 17, 9: 33, 17: 61, 18: 65, 19: 69}.items():
        assert pyconv.gaussmat(sigma, 0.2, True, "float")[0].shape == (1, n), sigma


# ------------------------------------------------------------------------------------------------ GPU: float, 1-D

@pytest.mark.gpu
@pytest.mark.parametrize("n,orient,family,seed", list(line_cases()))
def test_gpu_line_mask(vb, monkeypatch, n, orient, family, seed):
    """one 1-D mask on every kernel that can take it, on eight images: the oracle exactly, the float64 reference within
    tolerance"""
    m, scale, offset = line_mask(n, family, seed)
    mask = oriented(m, orient)
    for a in line_images(n, orient, seed):
        want = pyconv.conv(a, mask, scale, offset, "float")
        r, mag = ref64(a, mask, scale, offset)
        for kern, env in env_kernels(mask, scale).items():
            set_env(monkeypatch, env)
            got = vb.Image(a).conv(mask, scale, offset, "float").numpy()
            what = (kern, a.shape, a.dtype)
            same(got, want, what)
            within(got, r, mag, what)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", FORMATS)
def test_gpu_line_mask_every_format_and_band_count(vb, monkeypatch, dt):
    """each kernel's template instance for every format, at 1, 3 and 4 bands"""
    rng = np.random.default_rng(FORMATS.index(dt))
    masks = [line_mask(n, f, n) for n, f in ((9, "rand"), (16, "gauss"), (17, "sparse"), (64, "gauss"), (100, "spread"), (70, "rand"))]
    for b in BANDS:
        a = image(rng, dt, (29, 35, b), special=True)
        for m, scale, offset in masks:
            for orient in ("row", "col"):
                mask = oriented(m, orient)
                want = pyconv.conv(a, mask, scale, offset, "float")
                r, mag = ref64(a, mask, scale, offset)
                for kern, env in env_kernels(mask, scale).items():
                    set_env(monkeypatch, env)
                    got = vb.Image(a).conv(mask, scale, offset, "float").numpy()
                    same(got, want, (kern, b, m.size))
                    within(got, r, mag, (kern, b, m.size))


@pytest.mark.gpu
@pytest.mark.parametrize("sigma,kernel", [(4.5, "dense"), (9, "dense"), (17, "dense"), (18, "convf"), (19, "convf")])
def test_gpu_gaussblur_float_long_masks(vb, sigma, kernel):
    m, scale, _ = pyconv.gaussmat(sigma, 0.2, True, "float")
    assert expected_kernel(m, scale).startswith(kernel)
    rng = np.random.default_rng(int(sigma))
    for shape, dt in (((9, 150, 3), np.float32), ((150, 7, 1), np.uint8), ((5, 5, 4), np.uint16), ((40, 41, 3), np.int16)):
        a = image(rng, dt, shape)
        got = vb.Image(a).gaussblur(sigma, 0.2, "float").numpy()
        same(got, pyconv.gaussblur(a, sigma, 0.2, "float"), shape)
        within(got, *ref64_sep(a, m, scale), what=shape)


# ------------------------------------------------------------------------------------------------ GPU: float, 2-D and convsep

def masks_2d():
    rng = np.random.default_rng(5)
    out = []
    for sigma in (1.0, 2.0, 3.0, 4.5, 6.0):  # gaussmat 3 x 3, 7 x 7, 11 x 11, 17 x 17, 21 x 21, not separable
        m, scale, _ = pyconv.gaussmat(sigma, 0.2, False, "float")
        out.append(pytest.param(m, scale, 0.0, id="gauss%dx%d" % m.shape))
    for h, w in ((15, 3), (3, 15)):
        m = rng.uniform(-1, 1, (h, w))
        m[rng.random((h, w)) < 0.6] = 0
        out.append(pytest.param(m, -2.5, 1.25, id="sparse%dx%d" % (h, w)))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("mask,scale,offset", masks_2d())
def test_gpu_conv_2d(vb, mask, scale, offset):
    """convf_kernel with masks up to 21 x 21, including masks larger than the image"""
    assert expected_kernel(mask, scale) == "convf"
    rng = np.random.default_rng(mask.size)
    for i, shape in enumerate(((1, 1), (1, 37), (37, 1), (7, 9), (9, 7), (61, 83))):
        dt = FORMATS[(mask.size + i) % len(FORMATS)]
        a = image(rng, dt, shape + (BANDS[i % 3],), special=True)
        got = vb.Image(a).conv(mask, scale, offset, "float").numpy()
        same(got, pyconv.conv(a, mask, scale, offset, "float"), (shape, dt))
        within(got, *ref64(a, mask, scale, offset), what=(shape, dt))


SEP_LENGTHS = [1, 2, 3, 7, 8, 9, 15, 16, 17, 23, 24, 33, 64, 65, 66, 80, 129]


def sep_mask(n, family, seed, precision):
    m, scale, offset = line_mask(n, family, seed)
    if precision == "integer":
        m = np.rint(m * 20 / np.abs(m).max()) if m.any() else m
        s = m.sum()
        return m, (s if abs(s) >= 1 else 7.0), 3.0
    return m, scale, offset


@pytest.mark.gpu
@pytest.mark.parametrize("n", SEP_LENGTHS)
@pytest.mark.parametrize("orient", ["row", "col"])
@pytest.mark.parametrize("precision", ["float", "integer"])
def test_gpu_convsep(vb, monkeypatch, n, orient, precision):
    """the two passes of vips_convsep (first with the offset, then rot90 of the mask) on every kernel"""
    rng = np.random.default_rng(n)
    for fi, family in enumerate(("gauss", "rand", "head0", "tail0", "spread")):
        seed = n * 10 + fi
        m, scale, offset = sep_mask(n, family, seed, precision)
        mask = oriented(m, orient)
        envs = env_kernels(mask, scale) if precision == "float" else {"convi": "default"}
        for i, shape in enumerate(((61, 83), (7, 9), (1, 37), (37, 1))):
            dt = FORMATS[(seed + i) % len(FORMATS)]
            a = image(rng, dt, shape + (BANDS[(fi + i) % 3],))
            want = pyconv.convsep(a, mask, scale, offset, precision)
            for kern, env in envs.items():
                set_env(monkeypatch, env)
                got = vb.Image(a).convsep(mask, scale, offset, precision).numpy()
                same(got, want, (family, kern, shape, dt))
                if precision == "float":
                    within(got, *ref64_sep(a, mask, scale, offset), what=(family, kern, shape, dt))


@pytest.mark.gpu
def test_gpu_conv_device_input_with_padded_pitch(vb):
    """a device-resident input whose row pitch is padded by a multiple of the element size that is not a multiple of 16
    bytes: the dense kernel steps down a column by in_bpl / sizeof(T), the others by in_bpl"""
    torch = pytest.importorskip("torch")
    L = vb.lib()
    rng = np.random.default_rng(77)
    m17, s17, _ = line_mask(17, "gauss", 1)
    m9, s9, o9 = line_mask(9, "sparse", 2)
    m80, s80, o80 = line_mask(80, "spread", 3)
    cases = [(oriented(m17, "row"), s17, 0.0, "float"), (oriented(m17, "col"), s17, 0.0, "float"),
             (oriented(m9, "col"), s9, o9, "float"), (oriented(m80, "col"), s80, o80, "float"),
             (rng.uniform(-1, 1, (5, 5)), 1.5, 0.25, "float"), (np.rint(rng.uniform(-9, 9, (3, 3))), 5.0, 1.0, "integer")]
    assert [expected_kernel(m, s) for m, s, _, p in cases if p == "float"] == ["dense_h", "dense_v", "block_v", "line_v", "convf"]
    for dt, pad in ((np.uint8, 3), (np.int16, 3), (np.int32, 1), (np.float32, 3)):
        esize = np.dtype(dt).itemsize
        h, w, b = 37, 29, 3
        a = image(rng, dt, (h, w, b))
        line = w * b * esize
        pitch = line + pad * esize
        assert (pad * esize) % 16 and pitch % esize == 0
        buf = torch.zeros((h, pitch), dtype=torch.uint8, device="cuda")
        buf[:, :line] = torch.from_numpy(a.view(np.uint8).reshape(h, line)).cuda()
        for mask, scale, offset, precision in cases:
            odt = np.dtype(np.float32 if precision == "float" else dt)
            out = torch.empty((h, w * b * odt.itemsize), dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            cin = vb.CImage(w, h, b, vb.FORMATS[np.dtype(dt)], 22, vb.DEVICE, C.c_void_p(buf.data_ptr()), pitch)
            cout = vb.CImage(0, 0, 0, 0, 0, vb.DEVICE, C.c_void_p(out.data_ptr()), w * b * odt.itemsize)  # the result lands here
            m, cm = vb.Image._mask(mask, scale, offset)
            vb._check(L.vb200_conv(C.byref(cin), C.byref(cout), C.byref(cm), vb.PRECISIONS[precision]))
            torch.cuda.synchronize()
            assert cout.data == out.data_ptr() and cout.bpl == w * b * odt.itemsize
            got = out.cpu().numpy().view(odt).reshape(h, w, b)
            same(got, pyconv.conv(a, mask, scale, offset, precision), (dt, mask.shape, precision))


# ------------------------------------------------------------------------------------------------ GPU: integer precision

def extremes(rng, dt, shape):
    """pixels at both ends of the format's range, their neighbours, zero and random values"""
    dt = np.dtype(dt)
    if dt.kind == "f":
        a = ((rng.random(shape) - 0.5) * 2e6).astype(dt)
        big = np.finfo(np.float32).max / 1e6  # times 9 coefficients near 10^4 stays finite
        special = np.array([big, -big, 0.0, np.nan], dt)
        a.reshape(-1)[:min(4, a.size)] = special[:min(4, a.size)]
        return a
    i = np.iinfo(dt)
    pick = np.array([i.min, i.min + 1, 0, i.max - 1, i.max], np.int64)
    a = np.where(rng.random(shape) < 0.6, pick[rng.integers(0, 5, shape)],
                 rng.integers(i.min, int(i.max) + 1, shape, dtype=np.int64))
    return a.astype(dt)


def integer_masks():
    rng = np.random.default_rng(9)
    big = lambda shape: rng.integers(-12000, 12000, shape).astype(np.float64)  # a 32-bit sum of these overflows on int32 / uint32
    return [("3x3", big((3, 3)), 7.0, 0.0), ("1x9 negative scale", big((1, 9)), -3.0, 2.5),
            ("9x1 fractional", big((9, 1)), 2.5, -1.5), ("5x7 fractional", big((5, 7)), 3.5, 0.5),
            ("1x1", np.array([[10007.0]]), 1.0, 0.0), ("clip high", np.array([[1.0, 2.0, 1.0]]), 4.0, 70000.0),
            ("clip low", np.array([[1.0], [2.0], [1.0]]), 4.0, -70000.0), ("zero", np.zeros((3, 5)), 1.0, 1.0),
            ("small", np.rint(rng.uniform(-5, 5, (3, 3))), 1.0, 0.0)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", FORMATS)
def test_gpu_conv_integer_precision(vb, dt):
    """convi_kernel (int64 sums, (sum + scale / 2) / scale truncating, clip or wrap) and convi_float_kernel: every format at
    both ends of its range, coefficients near 10^4, negative and fractional scale and offset, offsets past both clips"""
    rng = np.random.default_rng(FORMATS.index(dt) + 30)
    for name, mask, scale, offset in integer_masks():
        for shape in ((23, 29, 3), (1, 1, 1), (5, 40, 4), (40, 2, 1)):
            a = extremes(rng, dt, shape)
            same(vb.Image(a).conv(mask, scale, offset, "integer").numpy(), pyconv.conv(a, mask, scale, offset, "integer"), (name, shape))


@pytest.mark.gpu
def test_gpu_conv_integer_scale_rounding_to_zero_is_refused(vb):
    a = np.zeros((4, 4, 1), np.uint8)
    with pytest.raises(ValueError):
        pyconv.conv(a, np.ones((3, 3)), 0.4, 0, "integer")
    with pytest.raises(vb.Error, match="scale rounds to zero"):
        vb.Image(a).conv(np.ones((3, 3)), 0.4, 0, "integer")


@pytest.mark.gpu
def test_gpu_conv_vector_mode_accepts_and_refuses(vb):
    """set_vector_convi(True): a uchar mask vips_convi_intize accepts takes the 8-bit-mantissa arithmetic; one it refuses
    (a range too wide for the mantissa, more than 1 024 points) falls back to the C path, as the oracle does"""
    gi, gs, _ = pyconv.gaussmat(1.2, 0.2, False, "integer")
    cases = [("accepted", gi, gs, 0.0, True), ("accepted, offset", np.array([[1.0, 2.0, 5.0, 2.0, 1.0]]), 11.0, -7.0, True),
             ("range too wide", np.array([[1.0, 200.0, 1.0]]), 1.0, 0.0, False),
             ("range too wide, negative", np.array([[-90.0], [300.0], [-90.0]]), 2.0, 3.0, False),
             ("33 x 33", np.ones((33, 33)), 1089.0, 0.0, False)]
    rng = np.random.default_rng(12)
    try:
        vb.set_vector_convi(True)
        for name, mask, scale, offset, accepted in cases:
            assert (pyconv.convi_intize8(mask, scale) is not None) == accepted, name
            for shape in ((40, 50, 3), (1, 1, 4), (3, 70, 1)):
                a = image(rng, np.uint8, shape)
                want = pyconv.conv(a, mask, scale, offset, "integer", vector=True)
                same(vb.Image(a).conv(mask, scale, offset, "integer").numpy(), want, (name, shape))
                if not accepted:
                    same(want, pyconv.conv(a, mask, scale, offset, "integer"), (name, shape))
    finally:
        vb.set_vector_convi(False)


# ------------------------------------------------------------------------------------------------ GPU: sharpen

def sharpen_images(rng, bands, r):
    out = []
    for h, w in ((1, 1), (2, 33), (33, 2), (31, 31), (32, 32), (33, 33), (max(1, r), max(1, r - 1))):
        out.append(("random", image(rng, np.uint8, (h, w, bands))))
        out.append(("photo", photo(rng, h, w, bands)))
    for h, w in ((1, 1), (33, 33), (max(1, r), 2)):
        for name, v in (("white", 255), ("black", 0)):
            out.append((name, np.full((h, w, bands), v, np.uint8)))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("bands", [3, 4])
@pytest.mark.parametrize("sigma,n", list(SHARPEN_SIGMAS.items()), ids=["%dtaps" % n for n in SHARPEN_SIGMAS.values()])
def test_gpu_sharpen_every_tap_count(vb, monkeypatch, sigma, n, bands):
    """sharpen_fused_kernel at each tap count it is instantiated for (one launch), and the unfused chain it stands for,
    on images smaller than the halo and at the 32 x 32 tile edges, random, smooth, white and black"""
    rng = np.random.default_rng(n * 10 + bands)
    for name, a in sharpen_images(rng, bands, n // 2):
        for kw in LUTS:
            want = pyconv.sharpen(a, "srgb", sigma=sigma, **kw)
            monkeypatch.delenv("VB200_NO_SHARPEN_FUSED", raising=False)
            n0 = vb.launch_count()
            got = vb.Image(a, "srgb").sharpen(sigma=sigma, **kw).numpy()
            assert vb.launch_count() - n0 == 1, ("not the fused kernel", name, a.shape)
            same(got, want, ("fused", name, a.shape, kw))
            monkeypatch.setenv("VB200_NO_SHARPEN_FUSED", "1")
            n0 = vb.launch_count()
            got = vb.Image(a, "srgb").sharpen(sigma=sigma, **kw).numpy()
            assert vb.launch_count() - n0 > 1, ("not the unfused chain", name, a.shape)
            same(got, want, ("unfused", name, a.shape, kw))


@pytest.mark.gpu
@pytest.mark.parametrize("bands", [3, 4])
@pytest.mark.parametrize("sigma", list(WIDE_SHARPEN_SIGMAS))
def test_gpu_sharpen_wider_than_the_fused_kernel(vb, sigma, bands):
    """17 and 21 taps: 8-bit sRGB takes the unfused chain by itself"""
    rng = np.random.default_rng(int(sigma) + bands)
    for a in (image(rng, np.uint8, (40, 50, bands)), photo(rng, 45, 38, bands), image(rng, np.uint8, (1, 1, bands)),
              image(rng, np.uint8, (5, 7, bands)), np.full((9, 9, bands), 255, np.uint8)):
        for kw in LUTS:
            n0 = vb.launch_count()
            got = vb.Image(a, "srgb").sharpen(sigma=sigma, **kw).numpy()
            assert vb.launch_count() - n0 > 1
            same(got, pyconv.sharpen(a, "srgb", sigma=sigma, **kw), (a.shape, kw))


def sharpen_batch(vb, d_in, in_stride, d_out, out_stride, n_frames, w, h, bands, sigma=0.5, kw=LUTS[0]):
    return vb.lib().vb200_sharpen_batch_device(d_in, in_stride, d_out, out_stride, n_frames, w, h, bands, sigma, kw["x1"], kw["y2"],
                                               kw["y3"], kw["m1"], kw["m2"])


@pytest.mark.gpu
def test_gpu_sharpen_wide_mask_refused_by_the_batched_paths(vb):
    """the batched sharpen and the thumbnail plan's sharpen stage have only the fused kernel: a 17-tap mask is an error"""
    torch = pytest.importorskip("torch")
    L = vb.lib()
    d = torch.zeros(2 * 20 * 16 * 4, dtype=torch.uint8, device="cuda")
    o = torch.zeros_like(d)
    assert sharpen_batch(vb, d.data_ptr(), 20 * 16 * 4, o.data_ptr(), 20 * 16 * 4, 2, 16, 20, 4, sigma=4.0) == -1
    assert b"at most 15 taps" in L.vb200_error_buffer()
    L.vb200_error_clear()
    plan = vb.ThumbnailPlan(64, 48, 3, 16)
    plan.set_sharpen(sigma=4.0)
    with pytest.raises(vb.Error, match="mask too wide"):
        plan.run_host(np.zeros((1, 48, 64, 3), np.uint8))
    plan.set_sharpen(sigma=0.5)  # the plan still works
    frames = photo(np.random.default_rng(3), 48, 64, 3)[None]
    assert np.array_equal(plan.run_host(frames)[0], pyconv.sharpen(orc.thumbnail_image(frames[0], 16), "srgb"))


@pytest.mark.gpu
@pytest.mark.parametrize("bands,w,h,pad", [(4, 37, 21, 12), (3, 31, 22, 5), (3, 16, 16, 0)])
def test_gpu_sharpen_batch_frame_strides(vb, bands, w, h, pad):
    """frames further apart than their size (4 bands: a multiple of 4 apart; 3 bands: any stride), and no frames at all"""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(bands * 100 + pad)
    frame = w * h * bands
    in_stride, out_stride = frame + pad, frame + 2 * pad + (bands == 3)
    n = 3
    frames = [photo(rng, h, w, bands) for _ in range(n)]
    host = np.zeros(n * in_stride, np.uint8)
    for i, f in enumerate(frames):
        host[i * in_stride:i * in_stride + frame] = f.reshape(-1)
    d = torch.from_numpy(host).cuda()
    o = torch.full((n * out_stride,), 7, dtype=torch.uint8, device="cuda")
    for sigma, kw in ((0.5, LUTS[0]), (3.5, LUTS[1])):
        torch.cuda.synchronize()
        vb._check(sharpen_batch(vb, d.data_ptr(), in_stride, o.data_ptr(), out_stride, n, w, h, bands, sigma, kw))
        torch.cuda.synchronize()
        got = o.cpu().numpy()
        for i, f in enumerate(frames):
            same(got[i * out_stride:i * out_stride + frame].reshape(h, w, bands), pyconv.sharpen(f, "srgb", sigma=sigma, **kw), (i, sigma))
            assert (got[i * out_stride + frame:(i + 1) * out_stride] == 7).all(), "wrote between frames"
    o.fill_(7)
    torch.cuda.synchronize()
    vb._check(sharpen_batch(vb, d.data_ptr(), in_stride, o.data_ptr(), out_stride, 0, w, h, bands))
    torch.cuda.synchronize()
    assert (o.cpu().numpy() == 7).all(), "n_frames = 0 wrote"

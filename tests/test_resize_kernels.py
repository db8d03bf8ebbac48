"""vips_resize's pixel arithmetic at every format, band count and kernel, down and up.

dev_resize (libvips_b200/csrc/resample_kernels.cu) sends a reduction through dev_reduce_chain: shrinkv / shrinkh box
averages by the integer part of the shrink, then reducev / reduceh with the residual (uchar in four forms, chosen by the
row length: staged and unstaged IDP.2A when it is a multiple of 4 bytes -- staged also needs a multiple of 16 -- the u8x4
kernel, the generic kernel; reduceh's RGBA form for 4 bands).  An enlargement is dev_resize_up (affine.cu):
zoom_kernel for integral nearest, affine_scale_kernel<T> for nearest / bilinear / bicubic, and for uchar RGBA bicubic
the separable shared-memory kernel (vertical scale >= 1) or the per-pixel one.

Three expectations:
  * the oracle (oracle/pyoracle.py) equals the reference's own resize.c pipeline under oracle/_ref on every input the
    GPU tests use (recorded in tests/golden/ref_results.json.gz for machines without the reference), so kernel ==
    oracle below means kernel == reference;
  * on smooth inputs the oracle and the kernels lie within a derived bound of a plain float64 model of the continuous
    operation (model_resize), which shares no code with the oracle -- and the bound is shown to catch a shifted
    output, the wrong lanczos, the wrong gap and the wrong upsize centre;
  * every GPU result equals the oracle bit for bit (NaN equal to NaN).
"""
import functools
import math
import os

import numpy as np
import pytest

from oracle import pyoracle as orc
from oracle import pyref

needs_ref = pytest.mark.skipif(not pyref.available(), reason="oracle/_ref not built")

FORMATS = [np.uint8, np.int8, np.uint16, np.int16, np.uint32, np.int32, np.float32]
INT_FORMATS = FORMATS[:-1]
BANDS = (1, 2, 3, 4, 5)
KERNELS = ["nearest", "linear", "cubic", "mitchell", "lanczos2", "lanczos3", "mks2013", "mks2021"]
DOWN_SCALES = (0.999, 0.9, 0.5, 0.37, 1 / 3, 0.11, "1/w")
UP_KERNELS = ("nearest", "linear", "cubic", "lanczos3")
UP_SCALES = (1.01, 1.5, 2.0, 3.7, 8.0, 16.3)
DEFAULT_TILES = (128, 128, 16, 1)
SUBSAMPLE_REFUSAL = "subsample step"


def fid(dt):
    return np.dtype(dt).name


# ------------------------------------------------------------------------------------------------ inputs

def noise(dt, shape, seed):
    """uniform over the whole range of an integer format; for float, [-75, 225)"""
    rng = np.random.default_rng(seed)
    dt = np.dtype(dt)
    if dt.kind == "f":
        return ((rng.random(shape) - 0.25) * 300).astype(dt)
    i = np.iinfo(dt)
    return rng.integers(i.min, int(i.max) + 1, shape, dtype=np.int64).astype(dt)


def span(dt):
    """(centre, amplitude) of the smooth inputs: inside the range with room for lanczos overshoot"""
    dt = np.dtype(dt)
    if dt.kind == "f":
        return 0.0, 100.0
    i = np.iinfo(dt)
    return (int(i.min) + int(i.max) + 1) / 2.0, (int(i.max) - int(i.min)) * 0.35


def smooth(dt, shape, seed, omega=0.25):
    """a sum of three cosines per band, angular frequencies at most omega per pixel on each axis, rounded to the format.
    Returns the image and (Gy, Gx): bounds on |d/dy| and |d/dx| of the continuous signal, in codes per pixel."""
    rng = np.random.default_rng(seed)
    h, w, b = shape
    mid, amp = span(dt)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    out = np.empty(shape)
    gy = gx = 0.0
    for z in range(b):
        a = rng.uniform(0.2, 1.0, 3)
        a /= a.sum()
        wy, wx = rng.uniform(-omega, omega, (2, 3))
        ph = rng.uniform(0, 2 * np.pi, 3)
        out[..., z] = mid + amp * sum(a[k] * np.cos(wy[k] * y + wx[k] * x + ph[k]) for k in range(3))
        gy, gx = max(gy, amp * float(np.abs(a * wy).sum())), max(gx, amp * float(np.abs(a * wx).sum()))
    if np.dtype(dt).kind != "f":
        out = np.rint(out)
    return out.astype(dt), (gy, gx)


def extremes(dt, kind, shape=(21, 26, 4)):
    """min / max fields of an integer format: constants, checkerboards and stripes of period p on either axis, one max
    pixel on a min field"""
    i = np.iinfo(dt)
    h, w, b = shape
    y, x = np.mgrid[0:h, 0:w]
    if kind == "min":
        m = np.zeros((h, w), bool)
    elif kind == "max":
        m = np.ones((h, w), bool)
    elif kind == "dot":
        m = np.zeros((h, w), bool)
        m[h // 2, w // 2] = True
    else:
        form, p = kind[:-1], int(kind[-1])
        m = {"check": (y // p + x // p) % 2 == 0, "rows": (y // p) % 2 == 0, "cols": (x // p) % 2 == 0}[form]
    return np.where(m[:, :, None], i.max, i.min).astype(dt) * np.ones((1, 1, b), dt)


EXTREME_KINDS = ["min", "max", "dot"] + ["%s%d" % (f, p) for f in ("check", "rows", "cols") for p in (1, 2, 3)]


def float_specials(kind, shape=(21, 26, 3)):
    rng = np.random.default_rng(77)
    h, w, b = shape
    y, x = np.mgrid[0:h, 0:w]
    if kind == "huge":
        return np.where(((y + x) % 2 == 0)[:, :, None], 3e38, -3e38).astype(np.float32) * np.ones((1, 1, b), np.float32)
    if kind == "denormal":
        return (rng.integers(-1000, 1000, shape) * np.float32(1e-42)).astype(np.float32)
    a = ((rng.random(shape) - 0.5) * 200).astype(np.float32)
    if kind == "inf":
        a[5, 7, 0], a[12, 20, 1], a[0, 0, 2] = np.inf, -np.inf, np.inf
    elif kind == "nan":
        a[5, 7, 0], a[h - 1, w - 1, 1] = np.nan, np.nan
    return a


FLOAT_SPECIALS = ("huge", "denormal", "inf", "nan")


# ------------------------------------------------------------------------------------------------ the cases

def down_scale(scale, shape):
    return 1.0 / shape[1] if scale == "1/w" else scale


def device_refuses(shape, hscale, vscale, kernel, gap):
    """dev_resize declines a nearest reduction whose resize.c would first subsample (resize.c:167-205)"""
    h, w = shape[:2]
    hscale, vscale = max(hscale, 1.0 / w), max(vscale, 1.0 / h)
    if kernel != "nearest" or hscale > 1.0 or vscale > 1.0:
        return False
    if gap < 1.0:
        xf, yf = math.floor(1.0 / hscale), math.floor(1.0 / vscale)
    else:
        tw, th = int(w * hscale + 0.5), int(h * vscale + 0.5)
        xf = math.floor(w / tw / gap) if tw > 0 else 1
        yf = math.floor(h / th / gap) if th > 0 else 1
    return xf > 1 or yf > 1


def down_cases(dt):
    """(name, image, resize arguments) for the reductions of one format"""
    out = []
    for b in BANDS:
        a = noise(dt, (43, 59, b), 100 + b)
        for k in KERNELS:
            for s in DOWN_SCALES:
                out.append(("grid-%db-%s-%s" % (b, k, s), a, dict(scale=down_scale(s, a.shape), kernel=k)))
    if dt == np.uint8:
        # reducev's uchar forms by row length: 64 columns x 1..5 bands is a multiple of 16 bytes (staged); 61 columns
        # with 4 bands a multiple of 4 (unstaged IDP.2A); others the generic kernel
        for w in (64, 61):
            for b in BANDS:
                a = noise(dt, (70, w, b), 200 + w + b)
                for k in ("lanczos3", "linear", "mks2021"):
                    for s in (0.5, 0.37, 0.11):
                        out.append(("row-%dx%d-%s-%s" % (w, b, k, s), a, dict(scale=s, kernel=k)))
    a = noise(dt, (47, 53, 3), 300)
    for hs, vs in ((0.5, 1.0), (1.0, 0.5), (0.3, 0.8), (0.8, 0.3), (0.11, 1.0), (1.0, 0.07)):
        for k in ("lanczos3", "cubic", "linear", "nearest"):
            out.append(("pair-%s-%s-%s" % (hs, vs, k), a, dict(scale=hs, vscale=vs, kernel=k)))
    for gap in (0.0, 1.0, 2.0, 3.3):
        for s in (0.5, 0.23, 0.11):
            for k in ("lanczos3", "mitchell", "linear"):
                out.append(("gap-%s-%s-%s" % (gap, s, k), a, dict(scale=s, kernel=k, gap=gap)))
    for h in (1, 2, 5, 17):
        for w in (1, 2, 5, 17):
            t = noise(dt, (h, w, 2), 400 + 31 * h + w)
            for k in ("lanczos3", "mks2021", "cubic", "linear"):
                for s in (0.9, 0.5, 0.3):
                    out.append(("tiny-%dx%d-%s-%s" % (h, w, k, s), t, dict(scale=s, kernel=k)))
    return out


def up_cases(dt):
    out = []
    for b in BANDS:
        a = noise(dt, (11, 13, b), 500 + b)
        for k in UP_KERNELS:
            for s in UP_SCALES:
                out.append(("grid-%db-%s-%s" % (b, k, s), a, dict(scale=s, kernel=k)))
    a = noise(dt, (9, 12, 3), 600)
    for k in UP_KERNELS:
        for s in (1.5, 3.7, 16.3):
            out.append(("axis-h-%s-%s" % (k, s), a, dict(scale=s, vscale=1.0, kernel=k)))
            out.append(("axis-v-%s-%s" % (k, s), a, dict(scale=1.0, vscale=s, kernel=k)))
    for shape in ((1, 1, 3), (1, 7, 3), (7, 1, 3)):
        t = noise(dt, shape, 700 + shape[0] * 10 + shape[1])
        for k in UP_KERNELS:
            out.append(("thin-%dx%d-%s" % (shape[0], shape[1], k), t, dict(scale=37.5, kernel=k)))
    for b in BANDS:
        a = noise(dt, (13, 17, b), 800 + b)
        for hs, vs in ((2, 2), (3, 7), (5, 1), (1, 4)):
            out.append(("zoom-%db-%dx%d" % (b, hs, vs), a, dict(scale=float(hs), vscale=float(vs), kernel="nearest")))
    return out


def extreme_cases(dt):
    out = []
    if np.dtype(dt).kind == "f":
        for kind in FLOAT_SPECIALS:
            a = float_specials(kind)
            for k in KERNELS:
                out.append(("%s-down-%s" % (kind, k), a, dict(scale=0.5, kernel=k)))
            for k in UP_KERNELS:
                out.append(("%s-up-%s" % (kind, k), a, dict(scale=2.5, kernel=k)))
        return out
    for kind in EXTREME_KINDS:
        a = extremes(dt, kind)
        for k in KERNELS:
            for s in (0.5, 0.37):
                out.append(("%s-down-%s-%s" % (kind, k, s), a, dict(scale=s, kernel=k)))
        for k in UP_KERNELS:
            for s in (2.0, 3.7):
                out.append(("%s-up-%s-%s" % (kind, k, s), a, dict(scale=s, kernel=k)))
    return out


def rgba_cases():
    """uchar RGBA bicubic enlargements: output sizes off the 64 x 32 tile grid, vscale 1 (a 32-row tile reads its whole
    35-row budget), just above 1, 2 and 4"""
    out = []
    for shape in ((45, 71), (77, 50), (33, 97)):
        a = noise(np.uint8, shape + (4,), 900 + shape[0])
        for hs in (1.7, 2.3):
            for vs in (1.0, 1.0001, 2.0, 4.0):
                out.append(("%dx%d-%s-%s" % (shape[0], shape[1], hs, vs), a, dict(scale=hs, vscale=vs, kernel="cubic")))
    return out


TILE_FORMATS = (np.int16, np.uint32, np.float32)
TILE_GEOMETRIES = ((64, 64), (10, 10), (512, 512))


def tile_cases(dt):
    """reductions whose rect heights / tile widths change the phase tables: box shrink and a residual"""
    a = noise(dt, (300, 257, 3), 1000)
    return [("%s-%s" % (s, k), a, dict(scale=s, kernel=k)) for s in (0.23, 0.37, 0.11) for k in ("lanczos3", "cubic")]


def run_oracle(a, kw, tile=(0, 0)):
    return orc.resize(a, kw["scale"], kw.get("vscale"), kernel=kw["kernel"], gap=kw.get("gap", 2.0), tile=tile)


def run_ref(a, kw, tile=(0, 0)):
    return pyref.RefImage.from_array(a).resize(kw["scale"], kw.get("vscale"), kernel=kw["kernel"],
                                               gap=kw.get("gap", 2.0)).numpy(tile=tile)


def run_device(vb, a, kw):
    return vb.Image(a).resize(kw["scale"], kw.get("vscale"), kernel=kw["kernel"], gap=kw.get("gap", 2.0)).numpy()


def refused(a, kw):
    vs = kw.get("vscale")
    return device_refuses(a.shape, kw["scale"], kw["scale"] if vs is None else vs, kw["kernel"], kw.get("gap", 2.0))


def same(got, want, what=""):
    """bit-exact, NaN equal to NaN"""
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    if not np.array_equal(got, want, equal_nan=got.dtype.kind == "f"):
        bad = got != want
        if got.dtype.kind == "f":
            bad &= ~(np.isnan(got) & np.isnan(want))
        raise AssertionError("%s: %d differ, first at %s: %s vs %s" % (what, bad.sum(), np.argwhere(bad)[:3].tolist(),
                                                                        got[bad][:3], want[bad][:3]))


def is_up(kw):
    vs = kw.get("vscale")
    return kw["scale"] > 1.0 or (kw["scale"] if vs is None else vs) > 1.0


def is_zoom(kw):
    vs = kw.get("vscale")
    vs = kw["scale"] if vs is None else vs
    hs = kw["scale"]
    return kw["kernel"] == "nearest" and hs >= 1 and vs >= 1 and hs * vs > 1 and hs == int(hs) and vs == int(vs)


def same_as_ref(a, kw, what, tile=(0, 0)):
    got = run_oracle(a, kw, tile)
    if is_zoom(kw):
        # vips_zoom (resize.c:263-271), which the reference build leaves out: every pixel an xfac x yfac block
        vs = kw["scale"] if kw.get("vscale") is None else kw["vscale"]
        want = np.repeat(np.repeat(a, int(vs), axis=0), int(kw["scale"]), axis=1)
        assert np.array_equal(got, want), what
        return
    want = run_ref(a, kw, tile)
    assert np.array_equal(got, want, equal_nan=got.dtype.kind == "f"), (what, pyref.difference(got, want))


# ------------------------------------------------------------------------------------------------ the float64 model

def kernel_fn(kernel, x):
    """the continuous kernels of vips_reduce: tent, Catmull-Rom (B, C = 0, 1/2), Mitchell-Netravali (1/3, 1/3),
    lanczos a = 2 and 3, and Costella's magic kernel sharp 2013 and 2021"""
    ax = np.abs(x)
    if kernel == "linear":
        return np.where(ax < 1, 1 - ax, 0.0)
    if kernel in ("cubic", "mitchell"):
        B, C = (0.0, 0.5) if kernel == "cubic" else (1 / 3, 1 / 3)
        near = ((12 - 9 * B - 6 * C) * ax ** 3 + (-18 + 12 * B + 6 * C) * ax ** 2 + (6 - 2 * B)) / 6
        far = ((-B - 6 * C) * ax ** 3 + (6 * B + 30 * C) * ax ** 2 + (-12 * B - 48 * C) * ax + (8 * B + 24 * C)) / 6
        return np.where(ax <= 1, near, np.where(ax <= 2, far, 0.0))
    if kernel in ("lanczos2", "lanczos3"):
        n = int(kernel[-1])
        return np.where(ax <= n, np.sinc(x) * np.sinc(x / n), 0.0)
    if kernel == "mks2013":
        return np.select([ax < 0.5, ax < 1.5, ax < 2.5],
                         [17 / 16 - 7 / 4 * ax ** 2, (4 * ax ** 2 - 11 * ax + 7) / 4, -((ax - 2.5) ** 2) / 8], 0.0)
    if kernel == "mks2021":
        return np.select([ax < 0.5, ax < 1.5, ax < 2.5, ax < 3.5, ax < 4.5],
                         [577 / 576 - 239 / 144 * ax ** 2, (140 * ax ** 2 - 379 * ax + 239) / 144,
                          -(24 * ax ** 2 - 113 * ax + 130) / 144, (4 * ax ** 2 - 27 * ax + 45) / 144,
                          -(4 * ax ** 2 - 36 * ax + 81) / 1152], 0.0)
    raise ValueError(kernel)


def reduce_weights(kernel, n, rs, f):
    """the n taps about a centre at fraction f past the tap n // 2 - 1/2 (reducev.cpp's window), normalised"""
    if kernel == "nearest":
        return np.ones(1)
    w = kernel_fn(kernel, (np.arange(n) - n // 2 - f + 0.5) / rs)
    return w / w.sum()


def reduce_matrix(size, shrink, kernel, gap, delta=0.0):
    """one axis of vips_reduce{v,h} as an (out, in) matrix: the box average by int_shrink (edge pixels repeated), then
    the kernel at the exact source position (o + 1/2) * residual - 1/2 - offset of output o, over n_point taps.
    delta moves every centre, for the outputs whose nearest tap is a tie."""
    g = orc.reduce_geometry(size, shrink, kernel, gap)
    k = g.int_shrink
    box = np.zeros((g.shrunk_size, size))
    for j in range(g.shrunk_size):
        for t in range(k):
            box[j, min(j * k + t, size - 1)] += 1.0 / k
    if g.n_point == 0:
        return box, g
    n, rs, m = g.n_point, g.residual, g.n_point // 2
    r = np.zeros((g.out_size, g.shrunk_size))
    for o in range(g.out_size):
        y = (o + 0.5) * rs - 0.5 - g.offset + delta
        py = math.floor(y)
        np.add.at(r[o], np.clip(py - m + np.arange(n), 0, g.shrunk_size - 1), reduce_weights(kernel, n, rs, y - py))
    return r @ box, g


def catmull_rom(t):
    return np.array([(-t ** 3 + 2 * t ** 2 - t) / 2, (3 * t ** 3 - 5 * t ** 2 + 2) / 2, (-3 * t ** 3 + 4 * t ** 2 + t) / 2,
                     (t ** 3 - t ** 2) / 2])


def up_matrix(size, scale, kernel, idx=None, delta=0.0):
    """one axis of vips_resize's enlargement: output x samples the input at u = x / scale - idx, idx = (1 - 1 / scale)
    / 2 (0 for nearest), edge pixels repeated; nearest takes floor(u), bilinear and Catmull-Rom the exact fraction.
    A scale of exactly 1 leaves the axis alone."""
    if scale == 1.0:
        return np.eye(size)
    out = int(scale * size + 0.5)
    if idx is None:
        idx = 0.0 if kernel == "nearest" else 0.5 * (1 - 1 / scale)
    m = np.zeros((out, size))
    for x in range(out):
        u = x / scale - idx + delta
        p = math.floor(u)
        t = u - p
        if kernel == "nearest":
            taps, w = [p], [1.0]
        elif kernel == "linear":
            taps, w = [p, p + 1], [1 - t, t]
        else:
            taps, w = [p - 1, p, p + 1, p + 2], catmull_rom(t)
        np.add.at(m[x], np.clip(taps, 0, size - 1), w)
    return m


def model_resize(a, scale, vscale=None, kernel="lanczos3", gap=2.0, idx=None, delta=(0.0, 0.0)):
    """vips_resize in float64 with no rounding: (Rv, Rh) applied as out = Rv a Rh^T per band"""
    h, w = a.shape[:2]
    vscale = scale if vscale is None else vscale
    hscale, vscale = max(scale, 1.0 / w), max(vscale, 1.0 / h)
    x = a.astype(np.float64)
    if hscale > 1.0 or vscale > 1.0:
        rv = up_matrix(h, vscale, kernel, idx, delta[0])
        rh = up_matrix(w, hscale, kernel, idx, delta[1])
        zoom = kernel == "nearest" and hscale == int(hscale) and vscale == int(vscale)
        if zoom:    # vips_zoom: exact replication
            rv = np.eye(h)[np.arange(int(h * vscale)) // int(vscale)]
            rh = np.eye(w)[np.arange(int(w * hscale)) // int(hscale)]
    else:
        rv = reduce_matrix(h, 1 / vscale, kernel, gap, delta[0])[0] if vscale < 1.0 else np.eye(h)
        rh = reduce_matrix(w, 1 / hscale, kernel, gap, delta[1])[0] if hscale < 1.0 else np.eye(w)
    return np.einsum("oy,yxb,px->opb", rv, x, rh)


def model_envelope(a, **kw):
    """the model's lowest and highest answer over centres moved by +-1e-8 pixel on either axis: a nearest tap exactly on
    a tie may go either way once the kernel's coordinate is built by repeated addition.  Clipped to the format's range,
    which the operation's cast imposes too."""
    runs = [model_resize(a, delta=(dy, dx), **kw) for dy in (-1e-8, 1e-8) for dx in (-1e-8, 1e-8)]
    lo, hi = np.min(runs, axis=0), np.max(runs, axis=0)
    if np.dtype(a.dtype).kind != "f":
        i = np.iinfo(a.dtype)
        top = i.max
        if a.dtype == np.uint32 and is_up(kw) and kw["kernel"] not in ("nearest", "linear"):
            top = 2 ** 31 - 1   # bicubic.cpp clips uint32 to INT_MAX
        lo, hi = np.clip(lo, i.min, top), np.clip(hi, i.min, top)
    return lo, hi


def model_error(got, env):
    lo, hi = env
    assert got.shape == lo.shape, (got.shape, lo.shape)
    g = got.astype(np.float64)
    return float(np.max(np.maximum(np.maximum(lo - g, g - hi), 0.0)))


# ------------------------------------------------------------------------------------------------ the bound
#
# The oracle differs from model_resize in three ways, each bounded from the pass's definition, never from its output.
#
#  1. Phase.  reducev / reduceh and bicubic look their coefficients up at the fraction rounded to 1/64
#     (VB200_TRANSFORM_SCALE): (int) (2 * 64 * f) rounded up to even, at most 1/128 of a source pixel from f.
#     Moving a filter's centre by d changes its output by sum_i w_i'(c) v_i d; since the weights sum to 1 this is
#     sum_j S_j (v_{j+1} - v_j) d with S_j the partial sums of w', so at most SLOPE * G * d, where G bounds the step
#     between neighbouring source pixels and SLOPE = max over c of sum_j |S_j| (slope_gain, computed from the model's
#     own weights).  G is the continuous signal's gradient times the box size, plus 1 for the rounding of the input
#     and 2 for the box averages' rounding.
#  2. 12-bit coefficients.  Integer formats use shorts (int) (w * 4096), truncated: the sum of |w_s - w| over the taps
#     (coef_error, over all 65 phases) times the largest |value| the pass reads bounds the change.  Float formats and
#     32-bit bicubic use the double coefficients and have no such term.
#  3. Rounding.  The unsigned fixed-point round (v + 2048) >> 12 of reduce, the 8-bit bicubic stages and bilinear's
#     12-bit sum moves a value by at most 0.5.  The signed one (templates.h signed_fixed_round) adds -2048 to a
#     negative sum and the arithmetic shift then floors, so a negative result lands 0.5 to 1.5 below its value: 1.5.
#     The box averages move it by at most 1 (C division truncates toward zero and uchar's multiplier 2^24 / k is
#     rounded down), the conversion of a double to a 32-bit integer by less than 1.  Float rounds at 2^-24 of
#     |value| per stored result.
#
# Errors already present in a pass's input pass through it scaled by the L1 norm of its weights.

PHASE = 1.0 / 128


def fixed_round_error(dt):
    return 1.5 if np.iinfo(dt).min < 0 else 0.5


def l1_and_slope(weights, h=1e-6):
    """(max over the fraction f of sum |w(f)|, max of sum_j |S_j| for the partial sums S_j of dw / df)"""
    l1 = slope = 0.0
    for f in np.linspace(0.0, 1.0, 257):
        l1 = max(l1, float(np.abs(weights(f)).sum()))
        d = (weights(f + h) - weights(f - h)) / (2 * h)
        slope = max(slope, float(np.abs(np.cumsum(d)[:-1]).sum()))
    return l1, slope


def coef_error(weights):
    """max over the 65 phases of sum |trunc(w * 4096) / 4096 - w|"""
    return max(float(np.abs(np.trunc(weights(t / 64) * 4096) / 4096 - weights(t / 64)).sum()) for t in range(65))


@functools.lru_cache(maxsize=None)
def reduce_stats(kernel, n, rs):
    """(L1, slope gain, 12-bit coefficient error) of a reduce's weights"""
    if kernel == "nearest":
        return 1.0, 0.0, 0.0
    wf = lambda f: reduce_weights(kernel, n, rs, f)    # noqa: E731
    return l1_and_slope(wf) + (coef_error(wf),)


@functools.lru_cache(maxsize=None)
def bicubic_stats():
    return l1_and_slope(catmull_rom) + (coef_error(catmull_rom),)


def down_pass_bound(dt, kernel, g, grad, m_in, e_in):
    """the error after one reduce pass of geometry g, given the input's gradient per original pixel, largest |value|
    and error"""
    is_int = np.dtype(dt).kind != "f"
    k = g.int_shrink
    e = e_in + (1.0 if is_int and k > 1 else 0.0)
    step = k * (grad + (1 if is_int else 0)) + (2 if is_int and k > 1 else 0)
    if g.n_point == 0:
        return e, step
    l1, slope, coef = reduce_stats(kernel, g.n_point, g.residual)
    e = l1 * e + slope * step * PHASE
    if is_int:
        e += coef * m_in + fixed_round_error(dt)
    else:
        e += 2.0 ** -23 * m_in * l1
    return e, l1 * step + 2 * e


def down_bound(a, grads, kw):
    """the bound for a reduction (both scales < 1) of a smooth input with gradients grads = (Gy, Gx)"""
    dt = a.dtype
    h, w = a.shape[:2]
    vs = kw.get("vscale", kw["scale"])
    vs = kw["scale"] if vs is None else vs
    hs, vs = max(kw["scale"], 1.0 / w), max(vs, 1.0 / h)
    gap = kw.get("gap", 2.0)
    m = float(np.abs(a.astype(np.float64)).max())
    e, gx = 0.0, grads[1]
    if vs < 1.0:
        gv = orc.reduce_geometry(h, 1 / vs, kw["kernel"], gap)
        e, _ = down_pass_bound(dt, kw["kernel"], gv, grads[0], m, 0.0)
        if gv.n_point:
            l1 = reduce_stats(kw["kernel"], gv.n_point, gv.residual)[0]
            m, gx = m * l1 + e, gx * l1 + 2 * e
    if hs < 1.0:
        gh = orc.reduce_geometry(w, 1 / hs, kw["kernel"], gap)
        e, _ = down_pass_bound(dt, kw["kernel"], gh, gx, m, e)
    return e


def up_bound(a, grads, kw):
    """the bound for an enlargement of a smooth input (affine.cu / interpolate.c / bicubic.cpp)"""
    dt = np.dtype(a.dtype)
    kernel = kw["kernel"]
    m = float(np.abs(a.astype(np.float64)).max())
    is_int = dt.kind != "f"
    g = sum(grads) + (2 if is_int else 0)
    if kernel == "nearest":
        return 0.0
    if kernel == "linear":
        if dt.itemsize <= 2 and is_int:
            # the fraction truncated to 1/4096, the four 12-bit weights (sum exactly 4096) each within 1/4096, one
            # round by (v + 2048) >> 12 whatever the sign
            return g / 4096 + 4 * g / 4096 + 0.5
        return 1.0 + 2.0 ** -50 * m if is_int else 2.0 ** -23 * m
    l1, slope, c = bicubic_stats()
    phase = slope * g * PHASE
    if dt.itemsize == 1:
        # two 12-bit stages: four horizontal sums rounded, then the vertical sum of those rounded
        r = fixed_round_error(dt)
        e1 = c * m + r
        return phase + l1 * e1 + c * (l1 * m + e1) + r
    if is_int:
        return phase + 1.0 + 2.0 ** -50 * m
    return phase + 2.0 ** -22 * m * l1


def bound(a, grads, kw):
    vs = kw.get("vscale")
    vs = kw["scale"] if vs is None else vs
    return up_bound(a, grads, kw) if kw["scale"] > 1.0 or vs > 1.0 else down_bound(a, grads, kw)


def smooth_cases(dt):
    """(name, image, gradients, resize arguments) on which the model's bound is asserted"""
    out = []
    a, g = smooth(dt, (41, 57, 3), 1100)
    for k in KERNELS:
        for s in DOWN_SCALES + ((0.5, 0.8), (1.0, 0.3), (0.3, 1.0)):
            if isinstance(s, tuple):
                kw = dict(scale=s[0], vscale=s[1], kernel=k)
            else:
                kw = dict(scale=down_scale(s, a.shape), kernel=k)
            if not refused(a, kw):
                out.append(("down-%s-%s" % (k, s), a, g, kw))
    for gap in (0.0, 1.0, 3.3):
        for s in (0.5, 0.23):
            out.append(("gap-%s-%s" % (gap, s), a, g, dict(scale=s, kernel="lanczos3", gap=gap)))
    u, gu = smooth(dt, (11, 13, 3), 1200, omega=0.6)
    for k in UP_KERNELS:
        for s in UP_SCALES + ((2.5, 1.0), (1.0, 3.7)):
            kw = dict(scale=s[0], vscale=s[1], kernel=k) if isinstance(s, tuple) else dict(scale=s, kernel=k)
            out.append(("up-%s-%s" % (k, s), u, gu, kw))
    return out


# ------------------------------------------------------------------------------------------------ 1. CPU: oracle == reference

@needs_ref
@pytest.mark.parametrize("dt", FORMATS, ids=fid)
@pytest.mark.parametrize("family", ["down", "up", "extremes", "smooth"])
def test_oracle_matches_reference(dt, family):
    """every input the GPU tests below compare with the oracle, through the reference's resize.c"""
    if family == "smooth":
        cases = [(n, a, kw) for n, a, _, kw in smooth_cases(dt)]
    else:
        cases = {"down": down_cases, "up": up_cases, "extremes": extreme_cases}[family](dt)
    for name, a, kw in cases:
        same_as_ref(a, kw, name)


@needs_ref
def test_oracle_matches_reference_rgba():
    for name, a, kw in rgba_cases():
        same_as_ref(a, kw, name)


@needs_ref
@pytest.mark.parametrize("dt", TILE_FORMATS, ids=fid)
@pytest.mark.parametrize("tile", TILE_GEOMETRIES, ids=str)
def test_oracle_matches_reference_tiles(dt, tile):
    """the reference's sink at another tile geometry: reducev's rect height and reduceh's tile width change the
    phase tables"""
    for name, a, kw in tile_cases(dt):
        same_as_ref(a, kw, name, tile=tile)


# ------------------------------------------------------------------------------------------------ 2. CPU: the model

def test_model_kernels_are_normalised_and_interpolating():
    """the model's own sanity: every kernel is 1 at 0 (to 1e-3 for the sharpened ones), and its integer-spaced samples
    sum to 1; Catmull-Rom reproduces a ramp"""
    for k in KERNELS[1:]:
        for f in (0.0, 0.25, 0.5):
            s = float(kernel_fn(k, np.arange(-6, 7) + f).sum())
            assert abs(s - 1) < 2e-2, (k, f, s)
    for t in (0.0, 0.3, 0.5, 0.9):
        c = catmull_rom(t)
        assert abs(c.sum() - 1) < 1e-15 and abs(c @ np.array([-1, 0, 1, 2]) - t) < 1e-15


@pytest.mark.parametrize("dt", FORMATS, ids=fid)
def test_oracle_within_model_bound(dt):
    for name, a, g, kw in smooth_cases(dt):
        got = run_oracle(a, kw)
        err, b = model_error(got, model_envelope(a, **kw)), bound(a, g, kw)
        assert err <= b, (name, err, b)


def mutation_input(dt=np.uint8, omega=1.0):
    """cosines at 0.3 and omega radians per pixel on each axis, 30 codes each around 128.  At omega = 1 (uchar) there
    is energy above a 0.5 reduction's output Nyquist frequency, where lanczos2 and lanczos3 differ most; at 0.6 (float,
    whose bound has no rounding terms) in the band where a box prefilter and a wider lanczos differ."""
    rng = np.random.default_rng(1300)
    y, x = np.mgrid[0:64, 0:80].astype(np.float64)
    ph = rng.uniform(0, 2 * np.pi, 4)
    v = 128 + 30 * (np.cos(0.3 * y + ph[0]) + np.cos(omega * y + ph[1]) + np.cos(0.3 * x + ph[2]) +
                    np.cos(omega * x + ph[3]))
    g = 30 * (0.3 + omega)
    if np.dtype(dt).kind != "f":
        v = np.rint(v)
    return v.astype(dt)[:, :, None], (g, g)


def test_bound_catches_a_shifted_output():
    a, g = mutation_input()
    for kw in (dict(scale=0.5, kernel="lanczos3"), dict(scale=0.37, kernel="cubic"), dict(scale=2.5, kernel="linear")):
        got = run_oracle(a, kw)
        env = model_envelope(a, **kw)
        assert model_error(got, env) <= bound(a, g, kw), kw
        for shifted in (np.roll(got, 1, axis=1), np.roll(got, 1, axis=0)):
            assert model_error(shifted, env) > bound(a, g, kw), kw


def test_bound_catches_the_wrong_lanczos():
    a, g = mutation_input()
    for s in (0.5, 0.37):
        got = run_oracle(a, dict(scale=s, kernel="lanczos2"))
        kw = dict(scale=s, kernel="lanczos3")
        assert model_error(run_oracle(a, kw), model_envelope(a, **kw)) <= bound(a, g, kw)
        assert model_error(got, model_envelope(a, **kw)) > bound(a, g, kw), s


def test_bound_catches_the_wrong_gap():
    a, g = mutation_input(np.float32, 0.6)
    for s in (0.25, 0.2):
        got = run_oracle(a, dict(scale=s, kernel="lanczos3", gap=0.0))
        kw = dict(scale=s, kernel="lanczos3", gap=2.0)
        assert model_error(run_oracle(a, kw), model_envelope(a, **kw)) <= bound(a, g, kw)
        assert model_error(got, model_envelope(a, **kw)) > bound(a, g, kw), s


def test_bound_catches_the_wrong_upsize_centre():
    a, g = mutation_input()
    for k in ("linear", "cubic"):
        for s in (2.0, 3.7):
            kw = dict(scale=s, kernel=k)
            got = run_oracle(a, kw)
            assert model_error(got, model_envelope(a, **kw)) <= bound(a, g, kw)
            assert model_error(got, model_envelope(a, idx=0.0, **kw)) > bound(a, g, kw), (k, s)


def test_constant_images_within_the_coefficient_bound():
    """a constant image stays constant for 8-bit formats.  Wider integer formats keep it only to within the truncated
    12-bit coefficients' deficit times the value (the reference's reducev.cpp:957 truncates), and uint32 bicubic
    enlargements clip at INT_MAX as bicubic.cpp does -- both asserted, so a change to either shows."""
    for dt in INT_FORMATS:
        for kind in ("min", "max"):
            a = extremes(dt, kind)
            v = a.flat[0]
            for name, _, kw in [c for c in extreme_cases(dt) if c[0].startswith(kind + "-")]:
                got = run_oracle(a, kw)
                if np.dtype(dt).itemsize == 1 or int(v) == 0:
                    assert (got == v).all(), name
                elif dt == np.uint32 and "-up-" in name and kw["kernel"] in ("cubic", "lanczos3"):
                    assert (got == 2 ** 31 - 1).all(), name
                else:
                    err = np.abs(got.astype(np.float64) - float(v)).max()
                    assert abs(model_error(got, model_envelope(a, **kw)) - err) <= 1e-9 * abs(float(v))
                    assert err <= bound(a, (0.0, 0.0), kw), (name, err)


# ------------------------------------------------------------------------------------------------ 3. GPU: kernel == oracle

def check_device(vb, name, a, kw):
    if refused(a, kw):
        with pytest.raises(vb.Error, match=SUBSAMPLE_REFUSAL):
            run_device(vb, a, kw)
        return
    same(run_device(vb, a, kw), run_oracle(a, kw), name)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", FORMATS, ids=fid)
def test_gpu_resize_down(vb, dt):
    cases = down_cases(dt)
    assert any(refused(a, kw) for _, a, kw in cases)
    for name, a, kw in cases:
        check_device(vb, name, a, kw)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", FORMATS, ids=fid)
def test_gpu_resize_up(vb, dt):
    for name, a, kw in up_cases(dt):
        check_device(vb, name, a, kw)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", FORMATS, ids=fid)
def test_gpu_resize_extremes(vb, dt):
    for name, a, kw in extreme_cases(dt):
        check_device(vb, name, a, kw)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", FORMATS, ids=fid)
def test_gpu_resize_within_model_bound(vb, dt):
    for name, a, g, kw in smooth_cases(dt):
        got = run_device(vb, a, kw)
        same(got, run_oracle(a, kw), name)
        err, b = model_error(got, model_envelope(a, **kw)), bound(a, g, kw)
        assert err <= b, (name, err, b)


@pytest.mark.gpu
@pytest.mark.parametrize("separable", [True, False], ids=["separable", "per-pixel"])
def test_gpu_rgba_bicubic(vb, separable):
    """VB200_NO_AFFINE_SEP is read on every call: unset, vscale >= 1 runs the separable kernel"""
    old = os.environ.pop("VB200_NO_AFFINE_SEP", None)
    try:
        if not separable:
            os.environ["VB200_NO_AFFINE_SEP"] = "1"
        for name, a, kw in rgba_cases():
            same(run_device(vb, a, kw), run_oracle(a, kw), name)
    finally:
        os.environ.pop("VB200_NO_AFFINE_SEP", None)
        if old is not None:
            os.environ["VB200_NO_AFFINE_SEP"] = old


@pytest.mark.gpu
@pytest.mark.parametrize("dt", TILE_FORMATS, ids=fid)
def test_gpu_tile_geometry(vb, dt):
    try:
        for tile in TILE_GEOMETRIES:
            vb.set_tile_geometry(*tile)
            for name, a, kw in tile_cases(dt):
                same(run_device(vb, a, kw), run_oracle(a, kw, tile=tile), "%s at %s" % (name, tile))
    finally:
        vb.set_tile_geometry(*DEFAULT_TILES)

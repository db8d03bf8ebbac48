"""ctypes loader for oracle/_ref/libvipsref.so: the reference's OWN source files
(libvips resample/*.c*, conversion/{pre,unpre}multiply.c, ...) compiled in place
under the GLib-free shim (oracle/ref_shim).  TEST INFRASTRUCTURE ONLY.

Pipelines are built lazily exactly like libvips does (build() per op, then a
sink pulls tiles through the generate() callbacks), so the rects each generate
function sees are the ones the real library would produce.

The reference's sources are not part of this repository, so where the library
has not been built every answer comes from tests/golden/ref_results.json.gz,
written by a run of the tests with the library present and VB200_REF_RECORD=1.
Each answer there is keyed by a digest of the call (function, arguments, input
pixels).  Scalars are stored whole; an array is stored as its shape, dtype and
a digest of its values, and comes back as a Recorded, which np.array_equal
compares with an array by that digest.  A call that was never recorded raises
KeyError.
"""
import ast
import atexit
import ctypes as C
import functools
import gzip
import hashlib
import json
import os
import threading

import numpy as np

from . import pyoracle

_HERE = os.path.dirname(os.path.abspath(__file__))
PATH = os.path.join(_HERE, "_ref", "libvipsref.so")
GOLDEN = os.path.join(os.path.dirname(_HERE), "tests", "golden", "ref_results.json.gz")
_LIB = None


def live():
    """the reference library itself is here (built from the reference's sources)"""
    return os.path.exists(PATH)


def available():
    return live() or os.path.exists(GOLDEN)


# ------------------------------------------------------------------ recorded answers
_RECORDED = None     # key -> encoded answer, from GOLDEN
_NEW = {}            # answers given by the live library under VB200_REF_RECORD
_DEPTH = threading.local()


def _canon(x):
    """a stable, content-based description of a call argument"""
    if isinstance(x, RefImage):
        return x.key
    if isinstance(x, np.ndarray):
        return ("array", x.dtype.str, x.shape, hashlib.sha256(np.ascontiguousarray(x).tobytes()).hexdigest())
    if isinstance(x, (list, tuple)):
        return tuple(_canon(v) for v in x)
    if isinstance(x, dict):
        return tuple(sorted((k, _canon(v)) for k, v in x.items()))
    if isinstance(x, (np.integer, np.floating)):
        x = x.item()
    if isinstance(x, type):
        return x.__name__
    if isinstance(x, (bool, int, float, str)) or x is None:
        return repr(x)
    raise TypeError("cannot key a reference call on %r" % (x,))


def _key(*parts):
    return hashlib.sha256(repr(_canon(parts)).encode()).hexdigest()[:20]


def values_digest(a):
    """digest of an array's shape and values, such that two arrays np.array_equal(..., equal_nan=True) agree on it"""
    f = np.asarray(a).astype(np.float64) + 0.0  # -0.0 == 0.0
    f[np.isnan(f)] = np.nan
    return hashlib.sha256(repr(f.shape).encode() + f.tobytes()).hexdigest()[:16]


class Recorded:
    """A recorded reference array: its shape, dtype and values_digest."""

    def __init__(self, dtype, shape, digest, has_nan):
        self.dtype, self.shape, self.digest, self.has_nan = np.dtype(dtype), tuple(shape), digest, has_nan
        self.ndim = len(self.shape)

    def __repr__(self):
        return "Recorded(%s, %s, %s)" % (self.dtype, self.shape, self.digest[:12])

    def __array_function__(self, func, types, args, kwargs):
        if func is not np.array_equal:
            return NotImplemented
        equal_nan = kwargs.get("equal_nan", args[2] if len(args) > 2 else False)
        ds = []
        for x in args[:2]:
            if isinstance(x, Recorded):
                if x.has_nan and not equal_nan:
                    return False
                ds.append(x.digest)
            else:
                x = np.asarray(x)
                if not equal_nan and x.dtype.kind in "fc" and np.isnan(x).any():
                    return False
                ds.append(values_digest(x))
        return ds[0] == ds[1]


def difference(a, b):
    """why np.array_equal(a, b) failed, for an assertion message: the largest difference of two arrays, or the digests
    when one side is a Recorded"""
    if isinstance(a, Recorded) or isinstance(b, Recorded):
        da = a.digest if isinstance(a, Recorded) else values_digest(a)
        db = b.digest if isinstance(b, Recorded) else values_digest(b)
        return "values digest %s != %s (the recorded reference keeps no pixels to compare)" % (da, db)
    return "max diff %g" % np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).max()


def _encode(v):
    """an array as "dtype shape nan digest", a tuple as a list, a scalar as its repr"""
    if isinstance(v, np.ndarray):
        nan = int(v.dtype.kind in "fc" and bool(np.isnan(v).any()))
        return "%s %s %d %s" % (v.dtype.str, ",".join(map(str, v.shape)), nan, values_digest(v))
    if isinstance(v, tuple):
        return [_encode(x) for x in v]
    if isinstance(v, (np.integer, np.floating)):
        v = v.item()
    return repr(v)


def _decode(e):
    if isinstance(e, list):
        return tuple(_decode(x) for x in e)
    parts = e.split(" ")
    if len(parts) == 4:
        dtype, shape, nan, digest = parts
        return Recorded(dtype, [int(n) for n in shape.split(",") if n], digest, nan == "1")
    if e in ("nan", "inf", "-inf"):
        return float(e)
    return ast.literal_eval(e)  # repr of an int / float / bool / None


def _save_new():
    old = {}
    if os.path.exists(GOLDEN):
        with gzip.open(GOLDEN, "rt") as f:
            old = json.load(f)
    old.update(_NEW)
    with gzip.GzipFile(GOLDEN, "wb", mtime=0) as f:
        f.write(json.dumps(old, sort_keys=True, separators=(",", ":")).encode())


def _answer(key, compute):
    """the reference's answer to the call named by key: computed when the library is here, recorded otherwise"""
    global _RECORDED
    depth = getattr(_DEPTH, "n", 0)
    if live():
        _DEPTH.n = depth + 1
        try:
            v = compute()
        finally:
            _DEPTH.n = depth
        if depth == 0 and os.environ.get("VB200_REF_RECORD"):
            if not _NEW:
                atexit.register(_save_new)
            _NEW[key] = _encode(v)
        return v
    if _RECORDED is None:
        with gzip.open(GOLDEN, "rt") as f:
            _RECORDED = json.load(f)
    if key not in _RECORDED:
        raise KeyError("no recorded reference answer for this call (%s); record it with oracle/_ref built and "
                       "VB200_REF_RECORD=1" % key)
    return _decode(_RECORDED[key])


def recorded(fn):
    """fn's answers come from the reference library when it is here, else from GOLDEN"""
    @functools.wraps(fn)
    def wrap(*args, **kw):
        return _answer(_key(fn.__qualname__, args, kw), lambda: fn(*args, **kw))
    return wrap


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(PATH)
        for name in ("ref_image_new_from_memory", "ref_shrinkv", "ref_shrinkh", "ref_reducev", "ref_reduceh",
                     "ref_resize", "ref_premultiply", "ref_unpremultiply", "ref_colour_op", "ref_colourspace",
                     "ref_conv", "ref_convsep", "ref_gaussblur", "ref_sharpen", "ref_gaussmat", "ref_affine",
                     "ref_cast", "ref_colourspace_build"):
            if hasattr(L, name):
                getattr(L, name).restype = C.c_void_p
        L.ref_error.restype = C.c_char_p
        L.ref_image_new_from_memory.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        L.ref_shrinkv.argtypes = [C.c_void_p, C.c_int, C.c_int]
        L.ref_shrinkh.argtypes = [C.c_void_p, C.c_int, C.c_int]
        L.ref_reducev.argtypes = [C.c_void_p, C.c_double, C.c_int, C.c_double]
        L.ref_reduceh.argtypes = [C.c_void_p, C.c_double, C.c_int, C.c_double]
        L.ref_resize.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_int, C.c_double]
        L.ref_premultiply.argtypes = [C.c_void_p, C.c_double, C.c_int]
        L.ref_unpremultiply.argtypes = [C.c_void_p, C.c_double, C.c_int]
        L.ref_image_write_to_memory.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        for f in ("ref_image_width", "ref_image_height", "ref_image_bands", "ref_image_format", "ref_image_dhint"):
            getattr(L, f).argtypes = [C.c_void_p]
        L.ref_reduce_make_mask.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double]
        L.vips_reduce_get_points.argtypes = [C.c_int, C.c_double]
        if hasattr(L, "ref_colourspace_build"):
            L.ref_colourspace_build.argtypes = [C.c_void_p, C.c_int, C.c_int]
            L.ref_cast.argtypes = [C.c_void_p, C.c_int, C.c_int]
        if hasattr(L, "ref_thumbnail_calculate_shrink"):
            L.ref_thumbnail_calculate_shrink.restype = None
            L.ref_thumbnail_calculate_shrink.argtypes = [C.c_int] * 6 + [C.POINTER(C.c_double)] * 2
            L.ref_thumbnail_find_jpegshrink.argtypes = [C.c_int] * 7
        _LIB = L
    return _LIB


class RefImage:
    """A lazy reference image (VipsImage* inside the shim)."""

    def __init__(self, handle, keep=(), key=None):
        if live() and not handle:
            raise ValueError("reference op failed: %s" % lib().ref_error().decode())
        self.h = handle
        self.keep = keep  # keep source arrays alive
        self.key = key    # the recipe: source pixels and ops, for recorded answers

    @staticmethod
    def from_array(a, interpretation=None):
        a = np.ascontiguousarray(a)
        if a.ndim == 2:
            a = a[:, :, None]
        if interpretation is None:
            interpretation = 1 if a.shape[2] < 3 else 22
        key = ("from_array", _canon(a), interpretation)
        if not live():
            return RefImage(None, (a,), key)
        h = lib().ref_image_new_from_memory(a.ctypes.data, a.shape[1], a.shape[0], a.shape[2],
                                            pyoracle.FMT[a.dtype], interpretation)
        return RefImage(h, (a,), key)

    def _op(self, name, *args):
        key = self.key + ((name,) + args,)
        return RefImage(getattr(lib(), name)(self.h, *args) if live() else None, (self,), key)

    def shrinkv(self, f, ceil=False):
        return self._op("ref_shrinkv", f, int(ceil))

    def shrinkh(self, f, ceil=False):
        return self._op("ref_shrinkh", f, int(ceil))

    def reducev(self, f, kernel="lanczos3", gap=0.0):
        return self._op("ref_reducev", float(f), pyoracle._k(kernel), float(gap))

    def reduceh(self, f, kernel="lanczos3", gap=0.0):
        return self._op("ref_reduceh", float(f), pyoracle._k(kernel), float(gap))

    def resize(self, scale, vscale=None, kernel="lanczos3", gap=2.0):
        return self._op("ref_resize", float(scale), float(scale if vscale is None else vscale),
                        pyoracle._k(kernel), float(gap))

    def subsample(self, xfac, yfac):
        """subsample.c: out(x, y) = in(x * xfac, y * yfac)"""
        if live():
            lib().ref_subsample.restype = C.c_void_p
            lib().ref_subsample.argtypes = [C.c_void_p, C.c_int, C.c_int]
        return self._op("ref_subsample", int(xfac), int(yfac))

    def premultiply(self, max_alpha=0.0, uchar=False):
        return self._op("ref_premultiply", float(max_alpha), int(uchar))

    def unpremultiply(self, max_alpha=0.0, uchar=False):
        return self._op("ref_unpremultiply", float(max_alpha), int(uchar))

    def _shape(self):
        L = lib()
        return (L.ref_image_height(self.h), L.ref_image_width(self.h), L.ref_image_bands(self.h))

    @property
    def shape(self):
        return _answer(_key(self.key, "shape"), self._shape)

    @property
    def dhint(self):
        return _answer(_key(self.key, "dhint"), lambda: lib().ref_image_dhint(self.h))

    def colourspace(self, space, source_space):
        """vips_colourspace_build over colourspace.c's route table, every step a real VipsColour object (colour.c build,
        vips_colour_gen, the converter's line function); alpha through cast.c / linear.c"""
        return self._op("ref_colourspace_build", pyoracle._space(space), pyoracle._space(source_space))

    def cast(self, dtype, shift=False):
        return self._op("ref_cast", pyoracle.FMT[np.dtype(dtype)], int(shift))

    def numpy(self, tile=(0, 0)):
        """The sink: pull the image through generate() tile by tile."""
        def sink():
            out = np.empty(self._shape(), pyoracle.DTYPE[lib().ref_image_format(self.h)])
            if lib().ref_image_write_to_memory(self.h, out.ctypes.data, tile[0], tile[1]):
                raise ValueError("reference evaluation failed: %s" % lib().ref_error().decode())
            return out
        return _answer(_key(self.key, "numpy", tuple(tile)), sink)


@recorded
def reduce_make_mask(kernel, n_point, shrink, x):
    c = np.zeros(n_point, np.float64)
    lib().ref_reduce_make_mask(c.ctypes.data, pyoracle._k(kernel), n_point, shrink, x)
    return c


@recorded
def reduce_get_points(kernel, shrink):
    return lib().vips_reduce_get_points(pyoracle._k(kernel), shrink)


@recorded
def thumbnail_image(a, width, height=None, size="both", tile=(0, 0)):
    """vips_thumbnail_build's pixel chain for an 8-bit sRGB / B_W image
    (thumbnail.c:827-902): [premultiply uchar] -> resize -> [unpremultiply uchar]."""
    h, w, b = a.shape
    hs, vs = thumbnail_calculate_shrink(w, h, width, height, size)      # the reference's own arithmetic
    im = RefImage.from_array(a)
    premul = (b == 2 or b >= 4) and hs != 1.0 and vs != 1.0
    if premul:
        im = im.premultiply(uchar=True)
    im = im.resize(1.0 / hs, 1.0 / vs)
    if premul:
        im = im.unpremultiply(uchar=True)
    return im.numpy(tile)


# ------------------------------------------------------------------ colour
@recorded
def colour_line(step, a):
    """Run the reference's own *_line function over an (n, 3) array."""
    step = pyoracle.STEPS[step] if isinstance(step, str) else step
    a = np.ascontiguousarray(a).reshape(-1, 3)
    assert a.dtype == pyoracle.STEP_IO[step][0], (a.dtype, step)
    out = np.empty((a.shape[0], 3 + pyoracle.STEP_BANDS.get(step, 0)), pyoracle.STEP_IO[step][1])
    L = lib()
    L.ref_colour_line.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    if L.ref_colour_line(step, a.ctypes.data, out.ctypes.data, a.shape[0]):
        raise ValueError("ref_colour_line")
    return out


@recorded
def colour_table(which):
    L = lib()
    L.ref_colour_table.restype = C.c_void_p
    n = C.c_int()
    p = L.ref_colour_table(which, C.byref(n))
    dt = np.int32 if which in (0, 2) else np.float32
    return np.frombuffer((C.c_uint8 * (n.value * 4)).from_address(p), dtype=dt).copy()


# ------------------------------------------------------------------ vips_thumbnail's size arithmetic
@recorded
def thumbnail_calculate_shrink(w, h, width, height=None, size="both", crop=0):
    """vips_thumbnail_calculate_shrink (thumbnail.c:412-466), the file-static function itself (ref_shim/ref_thumbnail.c)"""
    hs, vs = C.c_double(), C.c_double()
    lib().ref_thumbnail_calculate_shrink(w, h, width, width if height is None else height, pyoracle.SIZES[size], crop,
                                         C.byref(hs), C.byref(vs))
    return hs.value, vs.value


@recorded
def thumbnail_find_jpegshrink(w, h, width, height=None, size="both", crop=0, linear=False):
    """vips_thumbnail_find_jpegshrink (thumbnail.c:490-517)"""
    return int(lib().ref_thumbnail_find_jpegshrink(w, h, width, width if height is None else height, pyoracle.SIZES[size], crop,
                                                   int(linear)))


@recorded
def thumbnail_size_table(cases):
    """thumbnail_calculate_shrink's (hshrink, vshrink) and thumbnail_find_jpegshrink's shrink, without and with linear,
    for each (w, h, width, height, size) of cases: an (n, 4) float64 array"""
    return np.array([thumbnail_calculate_shrink(w, h, tw, th, size) +
                     (thumbnail_find_jpegshrink(w, h, tw, th, size), thumbnail_find_jpegshrink(w, h, tw, th, size, linear=True))
                     for (w, h, tw, th, size) in cases], np.float64)

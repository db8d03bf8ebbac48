"""Convolution bindings for the oracle and for oracle/_ref (the reference's own
convf.c / convi.c / gaussmat.c).  TEST INFRASTRUCTURE ONLY."""
import ctypes as C

import numpy as np

from . import pyoracle, pyref

PREC = {"integer": 0, "float": 1, "approximate": 2}


def _prec(p):
    return PREC[p] if isinstance(p, str) else int(p)


# ------------------------------------------------------------------ oracle
def gaussmat(sigma, min_ampl, separable=False, precision="integer"):
    L = pyoracle.lib()
    L.orc_gaussmat_size.argtypes = [C.c_double, C.c_double]
    L.orc_gaussmat.restype = C.c_double
    L.orc_gaussmat.argtypes = [C.c_double, C.c_double, C.c_int, C.c_int, C.c_void_p]
    n = L.orc_gaussmat_size(sigma, min_ampl)
    m = np.zeros((1 if separable else n, n), np.float64)
    scale = L.orc_gaussmat(sigma, min_ampl, int(separable), int(_prec(precision) != 1), m.ctypes.data)
    return m, scale, 0.0


def _out_dtype(dt, precision):
    if _prec(precision) == 1:
        return np.float64 if dt == np.float64 else np.float32
    return dt


def conv(a, mask, scale=1.0, offset=0.0, precision="float", vector=False):
    a, h, w, b, f = pyoracle._img(a)
    mask = np.ascontiguousarray(mask, np.float64)
    if mask.ndim == 1:
        mask = mask[None, :]
    out = np.empty((h, w, b), _out_dtype(a.dtype, precision))
    L = pyoracle.lib()
    L.orc_conv.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_double,
                           C.c_double, C.c_int, C.c_int, C.c_void_p]
    if L.orc_conv(a.ctypes.data, w, h, b, f, mask.ctypes.data, mask.shape[1], mask.shape[0], scale, offset,
                  _prec(precision), int(vector), out.ctypes.data):
        raise ValueError("conv")
    return out


def convsep(a, mask, scale=1.0, offset=0.0, precision="float", vector=False):
    """mask: 1-D (taken as n x 1, horizontal pass first) or 2-D with one dimension 1 (a column
    runs the vertical pass first, then the reversed row: vips_rot90)."""
    a, h, w, b, f = pyoracle._img(a)
    mask = np.ascontiguousarray(mask, np.float64)
    if mask.ndim == 1:
        mask = mask[None, :]
    out = np.empty((h, w, b), _out_dtype(a.dtype, precision))
    L = pyoracle.lib()
    L.orc_convsep2.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_double,
                               C.c_double, C.c_int, C.c_int, C.c_void_p]
    if L.orc_convsep2(a.ctypes.data, w, h, b, f, mask.ctypes.data, mask.shape[1], mask.shape[0], scale, offset,
                      _prec(precision), int(vector), out.ctypes.data):
        raise ValueError("convsep")
    return out


def gaussblur(a, sigma, min_ampl=0.2, precision="integer", vector=False):
    a, h, w, b, f = pyoracle._img(a)
    out = np.empty((h, w, b), a.dtype if sigma < 0.2 else _out_dtype(a.dtype, precision))
    L = pyoracle.lib()
    L.orc_gaussblur.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_int,
                                C.c_int, C.c_void_p]
    if L.orc_gaussblur(a.ctypes.data, w, h, b, f, sigma, min_ampl, _prec(precision), int(vector), out.ctypes.data):
        raise ValueError("gaussblur")
    return out


def sharpen(a, interpretation, sigma=0.5, x1=2.0, y2=10.0, y3=20.0, m1=0.0, m2=3.0):
    a, h, w, b, f = pyoracle._img(a)
    out = np.empty((h, w, b), a.dtype)
    L = pyoracle.lib()
    L.orc_sharpen.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int] + [C.c_double] * 6 + [C.c_void_p]
    if L.orc_sharpen(a.ctypes.data, w, h, b, f, pyoracle._space(interpretation), sigma, x1, y2, y3, m1, m2,
                     out.ctypes.data):
        raise ValueError("sharpen")
    return out


def convi_intize8(mask, scale):
    mask = np.ascontiguousarray(mask, np.float64).ravel()
    mant = np.zeros(mask.size, np.int16)
    pos = np.zeros(mask.size, np.int32)
    nnz, exp = C.c_int(), C.c_int()
    L = pyoracle.lib()
    L.orc_convi_intize8.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.POINTER(C.c_int),
                                    C.POINTER(C.c_int)]
    if L.orc_convi_intize8(mask.ctypes.data, mask.size, scale, mant.ctypes.data, pos.ctypes.data, C.byref(nnz),
                           C.byref(exp)):
        return None
    return mant[:nnz.value], pos[:nnz.value], exp.value


# --------------------------------------------------------------- reference
def _rl():
    L = pyref.lib()
    L.ref_matrix.restype = C.c_void_p
    L.ref_matrix.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double]
    L.ref_conv.restype = C.c_void_p
    L.ref_conv.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    L.ref_gaussmat.restype = C.c_void_p
    L.ref_gaussmat.argtypes = [C.c_double, C.c_double, C.c_int, C.c_int]
    L.ref_matrix_scale.restype = C.c_double
    L.ref_matrix_offset.restype = C.c_double
    L.ref_matrix_scale.argtypes = [C.c_void_p]
    L.ref_matrix_offset.argtypes = [C.c_void_p]
    L.ref_matrix_data.restype = C.c_void_p
    L.ref_matrix_data.argtypes = [C.c_void_p]
    return L


@pyref.recorded
def ref_conv(a, mask, scale=1.0, offset=0.0, precision="float", vector=False, tile=(0, 0)):
    L = _rl()
    mask = np.ascontiguousarray(mask, np.float64)
    if mask.ndim == 1:
        mask = mask[None, :]
    m = L.ref_matrix(mask.ctypes.data, mask.shape[1], mask.shape[0], scale, offset)
    im = pyref.RefImage.from_array(a)
    out = pyref.RefImage(L.ref_conv(im.h, m, _prec(precision), int(vector)), (im, mask))
    return out.numpy(tile)


@pyref.recorded
def ref_gaussmat(sigma, min_ampl, separable=False, precision="integer"):
    L = _rl()
    m = L.ref_gaussmat(sigma, min_ampl, int(separable), _prec(precision))
    if not m:
        raise ValueError("ref gaussmat")
    w, h = L.ref_image_width(m), L.ref_image_height(m)
    data = np.frombuffer((C.c_uint8 * (w * h * 8)).from_address(L.ref_matrix_data(m)), dtype=np.float64)
    return data.reshape(h, w).copy(), L.ref_matrix_scale(m), L.ref_matrix_offset(m)


@pyref.recorded
def ref_convsep(a, mask, scale=1.0, offset=0.0, precision="float", tile=(0, 0)):
    """vips_convsep through the reference's own convsep.c / conv.c / rot.c / convf.c / convi.c"""
    L = _rl()
    L.ref_convsep.restype = C.c_void_p
    L.ref_convsep.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    mask = np.ascontiguousarray(mask, np.float64)
    if mask.ndim == 1:
        mask = mask[None, :]
    m = L.ref_matrix(mask.ctypes.data, mask.shape[1], mask.shape[0], scale, offset)
    im = pyref.RefImage.from_array(a)
    return pyref.RefImage(L.ref_convsep(im.h, m, _prec(precision)), (im, mask)).numpy(tile)


@pyref.recorded
def ref_sharpen(a, interpretation, sigma=0.5, x1=2.0, y2=10.0, y3=20.0, m1=0.0, m2=3.0, tile=(0, 0)):
    """vips_sharpen through the reference's own sharpen.c (build + generate), 3-band images"""
    L = _rl()
    L.ref_sharpen.restype = C.c_void_p
    L.ref_sharpen.argtypes = [C.c_void_p] + [C.c_double] * 6
    im = pyref.RefImage.from_array(a, pyoracle._space(interpretation))
    return pyref.RefImage(L.ref_sharpen(im.h, sigma, x1, y2, y3, m1, m2), (im,)).numpy(tile)


@pyref.recorded
def ref_sharpen_lut(sigma=0.5, x1=2.0, y2=10.0, y3=20.0, m1=0.0, m2=3.0):
    L = _rl()
    L.ref_sharpen_lut.argtypes = [C.c_double] * 6 + [C.c_void_p]
    lut = np.zeros(65536, np.int32)
    if L.ref_sharpen_lut(sigma, x1, y2, y3, m1, m2, lut.ctypes.data):
        raise ValueError("ref sharpen lut")
    return lut


def sharpen_lut(x1=2.0, y2=10.0, y3=20.0, m1=0.0, m2=3.0):
    L = pyoracle.lib()
    L.orc_sharpen_lut.argtypes = [C.c_double] * 5 + [C.c_void_p]
    lut = np.zeros(65536, np.int32)
    L.orc_sharpen_lut(x1, y2, y3, m1, m2, lut.ctypes.data)
    return lut


# ------------------------------------------------------------------ morphology
def morph(a, mask, op):
    """vips_morph, oracle restatement (uchar images; op "erode" / "dilate")"""
    a, h, w, b, f = pyoracle._img(a)
    assert a.dtype == np.uint8
    mask = np.ascontiguousarray(mask, np.float64)
    out = np.empty_like(a)
    L = pyoracle.lib()
    L.orc_morph.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    if L.orc_morph(a.ctypes.data, w, h, b, mask.ctypes.data, mask.shape[1], mask.shape[0], {"erode": 0, "dilate": 1}[op],
                   out.ctypes.data):
        raise ValueError("morph: bad mask element")
    return out


@pyref.recorded
def ref_morph(a, mask, op, tile=(0, 0)):
    """vips_morph through the reference's own morph.c (C generate functions)"""
    L = _rl()
    L.ref_morph.restype = C.c_void_p
    L.ref_morph.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    mask = np.ascontiguousarray(mask, np.float64)
    m = L.ref_matrix(mask.ctypes.data, mask.shape[1], mask.shape[0], 1.0, 0.0)
    im = pyref.RefImage.from_array(a)
    return pyref.RefImage(L.ref_morph(im.h, m, {"erode": 0, "dilate": 1}[op]), (im, mask)).numpy(tile)


def rank(a, width, height, index):
    """vips_rank, oracle restatement: the index-th smallest of each width x height window, per band"""
    a, h, w, b, f = pyoracle._img(a)
    out = np.empty_like(a)
    L = pyoracle.lib()
    L.orc_rank.argtypes = [C.c_void_p] + [C.c_int] * 7 + [C.c_void_p]
    if L.orc_rank(a.ctypes.data, w, h, b, f, width, height, index, out.ctypes.data):
        raise ValueError("rank: bad window, index or format")
    return out


def median(a, size):
    """vips_median, rank.c:651-664"""
    return rank(a, size, size, (size * size) // 2)


@pyref.recorded
def ref_rank(a, width, height, index, tile=(0, 0)):
    """vips_rank through the reference's own morphology/rank.c"""
    L = _rl()
    L.ref_rank.restype = C.c_void_p
    L.ref_rank.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    im = pyref.RefImage.from_array(a)
    return pyref.RefImage(L.ref_rank(im.h, width, height, index), (im,)).numpy(tile)


@pyref.recorded
def ref_flatten(a, background=(0.0,), max_alpha=0.0, interpretation=None, tile=(0, 0)):
    """vips_flatten through the reference's own conversion/flatten.c (+ cast.c for the ink and the double detour)"""
    L = _rl()
    L.ref_flatten.restype = C.c_void_p
    L.ref_flatten.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_double]
    bg = np.ascontiguousarray(background, np.float64)
    im = pyref.RefImage.from_array(a, interpretation)
    return pyref.RefImage(L.ref_flatten(im.h, bg.ctypes.data, len(bg), max_alpha), (im, bg)).numpy(tile)


def flatten(a, background=(0.0,), max_alpha=0.0, interpretation=None):
    """vips_flatten, oracle restatement.  interpretation: VipsInterpretation value (default as pyref: B_W / sRGB by bands)"""
    a, h, w, b, f = pyoracle._img(a)
    if interpretation is None:
        interpretation = 1 if b < 3 else 22
    bg = np.ascontiguousarray(background, np.float64)
    out = np.empty((h, w, max(1, b - 1)), a.dtype)
    L = pyoracle.lib()
    L.orc_flatten.argtypes = [C.c_void_p] + [C.c_int] * 5 + [C.c_void_p, C.c_int, C.c_double, C.c_void_p]
    rc = L.orc_flatten(a.ctypes.data, w, h, b, f, interpretation, bg.ctypes.data, len(bg), max_alpha, out.ctypes.data)
    if rc == -2:
        raise NotImplementedError("flatten: the reference's arithmetic is undefined here")
    if rc:
        raise ValueError("flatten: bad arguments")
    return out

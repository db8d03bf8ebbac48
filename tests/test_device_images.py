"""Device-resident images through every whole-image op of the C ABI: padded pitches, off-grid bases and caller buffers.

A VB200Image with where = VB200_DEVICE is read where it lies: its data and bpl reach the kernels as they are, and conv,
colourspace and the ICC ops write straight into a caller's out->data / out->bpl.  The layout therefore chooses the
kernel: the vector kernels run only on rows and bases that sit on a 4- or 16-byte grid.  Every op below runs over every
format it takes on the device path, in each of these input layouts, against the oracle (pyoracle / pyconv bit for bit;
ICC against the host evaluation vb200_debug_icc_eval within test_icc.py's bounds):

  packed   bpl = line, the buffer's base (256-byte aligned)
  padded   bpl = line + 3 elements: 3 bytes (off the 4-byte grid) for uchar / char, 6 or 12 bytes (off the 16-byte grid)
  offset   base + one element, padded bpl
  word     uchar / char: base + 4, bpl = line + 4 -- on the 4-byte grid, off the 16-byte one
  byteN    uchar / char with 3 or 4 bands: base + N (N = 1, 2, 3), bpl = line + 1

Input pitch padding holds a sentinel, so a kernel that read it would give other pixels.  VECTOR_PATHS is the table of
which side of each vector kernel's dispatch condition a layout lands on (mirroring the C conditions); VECTOR_CASES puts
every one of those kernels on both sides, with the non-layout half of each condition too (vshrink 257 / 258, ne % 4,
width % 4, a 4-band sharpen on and off the word grid).
"""
import ctypes as C
import zlib

import numpy as np
import pytest

import icc_fixtures as F
import libvips_b200 as vb
from oracle import pyconv
from oracle import pyoracle as orc

FORMATS = [np.uint8, np.int8, np.uint16, np.int16, np.uint32, np.int32, np.float32]
B_W, XYZ, LAB, CMYK, LABS, SRGB, RGB16 = 1, 12, 13, 15, 21, 22, 25
SPACE = {"b-w": B_W, "xyz": XYZ, "lab": LAB, "labs": LABS, "srgb": SRGB, "rgb16": RGB16, "scrgb": 28}
SENTINEL = 0xA5
TAIL = 40  # bytes after the last row of every buffer, all SENTINEL
SHAPES = ((29, 37), (3, 5))  # (height, width): ragged, and smaller than any tile
LANCZOS3 = 5


# ------------------------------------------------------------------------------------------------ layouts and buffers

def layouts(dt, bands):
    names = ["packed", "padded", "offset"]
    if np.dtype(dt).itemsize == 1:
        names.append("word")
        if bands in (3, 4):
            names += ["byte1", "byte2", "byte3"]
    return names


def placement(layout, dt, w, bands):
    """(byte offset of the base from the buffer's start, bpl) of a layout"""
    es = np.dtype(dt).itemsize
    line = w * bands * es
    if layout == "packed":
        return 0, line
    if layout == "padded":
        return 0, line + 3 * es
    if layout == "offset":
        return es, line + 3 * es
    if layout == "word":
        return 4, line + 4
    assert layout.startswith("byte")
    return int(layout[4:]), line + 1


class Buf:
    """h rows of `line` bytes at byte `off` of a buffer with stride bpl, on the device (a torch tensor) or the host (numpy).
    The pitch padding, the bytes before the base and a tail of TAIL bytes hold SENTINEL."""

    def __init__(self, h, line, off, bpl, rows=None, host=False):
        import torch
        self.h, self.line, self.off, self.bpl = h, line, off, bpl
        b = np.full(off + h * bpl + TAIL, SENTINEL, np.uint8)
        if rows is not None:
            self.body(b)[:] = np.ascontiguousarray(rows).view(np.uint8).reshape(h, line)
        self.host = host
        if host:
            self.np = b
            self.ptr = b.ctypes.data + off
        else:
            self.t = torch.from_numpy(b).cuda()
            assert self.t.data_ptr() % 256 == 0
            self.ptr = self.t.data_ptr() + off

    def body(self, b):
        return b[self.off:self.off + self.h * self.bpl].reshape(self.h, self.bpl)[:, :self.line]

    def bytes(self):
        import torch
        torch.cuda.synchronize()
        return self.np.copy() if self.host else self.t.cpu().numpy()

    def rows(self, dt, w, bands):
        return np.ascontiguousarray(self.body(self.bytes())).view(dt).reshape(self.h, w, bands)

    def assert_outside_untouched(self, what):
        b = self.bytes()
        outside = np.ones(b.size, bool)
        self.body(outside)[:] = False
        assert (b[outside] == SENTINEL).all(), (what, "wrote outside the rows", np.flatnonzero(b[outside] != SENTINEL)[:8])


def fmt_of(dt):
    return vb.FORMATS[np.dtype(dt)]


def device_image(a, layout, interp):
    h, w, b = a.shape
    off, bpl = placement(layout, a.dtype, w, b)
    buf = Buf(h, w * b * a.itemsize, off, bpl, a)
    return vb.CImage(w, h, b, fmt_of(a.dtype), interp, vb.DEVICE, C.c_void_p(buf.ptr), bpl), buf


class _DevPtr:
    """a raw device pointer seen by torch.as_tensor (the CUDA array interface)"""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 3, "strides": None}


def take_device(cout):
    """the pixels of a library-allocated device result, then vb200_image_free"""
    import torch
    assert cout.where == vb.DEVICE and cout.data
    dt = vb.DTYPES[cout.BandFmt]
    line = cout.Xsize * cout.Bands * np.dtype(dt).itemsize
    assert cout.bpl >= line
    torch.cuda.synchronize()
    b = torch.as_tensor(_DevPtr(cout.data, cout.Ysize * cout.bpl), device="cuda").cpu().numpy()
    vb.lib().vb200_image_free(C.byref(cout))
    assert cout.data is None
    return np.ascontiguousarray(b.reshape(cout.Ysize, cout.bpl)[:, :line]).view(dt).reshape(cout.Ysize, cout.Xsize, cout.Bands)


def same(got, want, what=""):
    """bit for bit, NaN equal to NaN"""
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    bad = got != want
    if got.dtype.kind == "f":
        bad &= ~(np.isnan(got) & np.isnan(want))
    assert not bad.any(), (what, int(bad.sum()), np.argwhere(bad)[:4], got[bad][:4], want[bad][:4])


def host_eval(mode, a, pa, pb=None, depth=8, pcs=0, intent=1):
    """vb200_debug_icc_eval: the ICC evaluator's per-pixel code on the CPU over packed pixels"""
    L = vb.lib()
    a = np.ascontiguousarray(a)
    n = a.size // a.shape[-1]
    out = np.zeros((n, 8), np.float32 if mode == 0 else (np.uint8 if depth == 8 else np.uint16))
    ob = L.vb200_debug_icc_eval(mode, a.ctypes.data, fmt_of(a.dtype), a.shape[-1], out.ctypes.data, n, pa, len(pa), pb,
                                len(pb) if pb else 0, intent, depth, pcs)
    if ob < 0:
        raise vb.Error(L.vb200_error_buffer().decode(errors="replace"))
    return np.ascontiguousarray(out.reshape(-1)[:n * ob].reshape(n, ob))


# ------------------------------------------------------------------------------------------------ inputs

def pixels(rng, dt, shape):
    """the whole range of an integer format; floats in [-20, 280)"""
    dt = np.dtype(dt)
    if dt.kind == "f":
        return (rng.random(shape) * 300 - 20).astype(dt)
    i = np.iinfo(dt)
    return rng.integers(i.min, int(i.max) + 1, shape, dtype=np.int64).astype(dt)


def colour_sample(space):
    def make(rng, dt, shape):
        h, w, b = shape
        if space in ("srgb", "b-w"):
            a = rng.integers(0, 256, shape, dtype=np.uint8)
        elif space == "rgb16":
            a = rng.integers(0, 65536, shape, dtype=np.uint16)
        elif space == "labs":
            a = rng.integers(-32768, 32768, shape, dtype=np.int64).astype(np.int16)
            a[..., 0] = np.abs(a[..., 0])
        elif space == "xyz":
            a = (rng.random(shape) * 110 - 5).astype(np.float32)
        else:  # lab
            a = rng.random(shape).astype(np.float32)
            a[..., 0] *= 100
            a[..., 1:3] = a[..., 1:3] * 256 - 128
        if b > 3 and a.dtype == np.float32:
            a[..., 3:] = rng.random((h, w, b - 3)) * 255
        return a
    return make


def host_lab(rng, dt, shape):
    """Lab floats as vips_icc_import makes them from random 8-bit sRGB"""
    h, w, _ = shape
    rgb = rng.integers(0, 256, (h * w, 3), dtype=np.uint8)
    return host_eval(0, rgb, F.rgb_profile()).reshape(h, w, 3).astype(np.float32)


# ------------------------------------------------------------------------------------------------ the ops

class Op:
    """call(L, in, out) -> rc; want(a) the oracle's array, or check(got, a) for a tolerance; in_place: the result fits
    in the input (same format, no larger)"""

    def __init__(self, name, formats, call, want=None, bands=(3, 4), interp=None, make=pixels, check=None, in_place=False,
                 out_type=None):
        self.name, self.formats, self.call, self.want, self.bands = name, formats, call, want, bands
        self.interp, self.make, self.in_place, self.out_type = interp, make, in_place, out_type
        self.check = check or (lambda got, a, what: same(got, self.want(a), what))

    def interp_for(self, bands):
        return self.interp if self.interp is not None else (SRGB if bands >= 3 else B_W)

    def expect(self, a):
        """shape and dtype of the result"""
        if self.want is not None:
            w = self.want(a)
            return w.shape, w.dtype
        return self.expect_fn(a)


def _mask_call(fn, mask, scale, offset, *extra):
    def call(L, i, o):
        m, cm = vb.Image._mask(mask, scale, offset)
        return getattr(L, fn)(i, o, C.byref(cm), *extra)
    return call


FLATTEN_BG = (10.7, 200.2, 33.0)


def flatten_max_alpha(dt):
    """the interpretation's default (255), but below char's range for char: there the reference's arithmetic at 255 is
    undefined C and the device path declines"""
    return 100.0 if np.dtype(dt) == np.int8 else 0.0


def _flatten_call(L, i, o):
    bg = np.array(FLATTEN_BG, np.float64)
    return L.vb200_flatten(i, o, bg.ctypes.data_as(C.c_void_p), len(bg), flatten_max_alpha(vb.DTYPES[i._obj.BandFmt]))


M33 = np.array([[0.25, -0.5, 0.125], [1.0, 0.75, -0.25], [0.0, 0.5, 0.375]])
MI33 = np.array([[1.0, -2.0, 3.0], [2.0, 5.0, -1.0], [0.0, 4.0, 1.0]])
SEP5 = np.array([[1.0, 4.0, 6.0, 4.0, 1.0]])
CROSS = np.array([[128.0, 255.0, 128.0], [255.0, 255.0, 0.0], [128.0, 255.0, 128.0]])
U8 = [np.uint8]


def _colour_op(src, dst, dt, bands):
    return Op("colour_%s_%s" % (src, dst), [dt], lambda L, i, o: L.vb200_colourspace(i, o, SPACE[dst]),
              lambda a: orc.colourspace(a, dst, src), bands=bands, interp=SPACE[src], make=colour_sample(src), out_type=SPACE[dst])


def _icc_within(want_fn, float_tol=2e-3):
    def check(got, a, what):
        want = want_fn(a).reshape(got.shape)
        assert got.dtype == want.dtype, (what, got.dtype, want.dtype)
        d = np.abs(got.astype(np.float64) - want.astype(np.float64))
        if got.dtype.kind == "f":
            assert d.max() < float_tol, (what, d.max())
        else:
            assert d.max() <= 1 and (d > 0).mean() < 2e-3 + 1.0 / d.size, (what, d.max(), (d > 0).mean())
    return check


def _icc_ops():
    rgb, ink = F.rgb_profile(), F.ink_profile()
    ops = []
    op = Op("icc_import_uchar", U8, lambda L, i, o: L.vb200_icc_import(i, o, rgb, len(rgb), 1, 0), bands=(3,), interp=SRGB,
            check=_icc_within(lambda a: host_eval(0, a.reshape(-1, 3), rgb)), out_type=LAB)
    op.expect_fn = lambda a: (a.shape, np.dtype(np.float32))
    ops.append(op)
    op = Op("icc_import_ushort", [np.uint16], lambda L, i, o: L.vb200_icc_import(i, o, ink, len(ink), 1, 1), bands=(4,),
            interp=CMYK, check=_icc_within(lambda a: host_eval(0, a.reshape(-1, 4), ink, pcs=1)), out_type=XYZ)
    op.expect_fn = lambda a: (a.shape[:2] + (3,), np.dtype(np.float32))
    ops.append(op)
    op = Op("icc_export_float", [np.float32], lambda L, i, o: L.vb200_icc_export(i, o, rgb, len(rgb), 1, 8, 0), bands=(3,),
            interp=LAB, make=host_lab, check=_icc_within(lambda a: host_eval(1, a.reshape(-1, 3), rgb)), out_type=SRGB)
    op.expect_fn = lambda a: (a.shape, np.dtype(np.uint8))
    ops.append(op)
    op = Op("icc_transform_uchar", U8, lambda L, i, o: L.vb200_icc_transform(i, o, rgb, len(rgb), ink, len(ink), 1, 8),
            bands=(3,), interp=SRGB, check=_icc_within(lambda a: host_eval(2, a.reshape(-1, 3), rgb, ink)), out_type=CMYK)
    op.expect_fn = lambda a: (a.shape[:2] + (4,), np.dtype(np.uint8))
    ops.append(op)
    return ops


OPS = [
    Op("shrinkv", FORMATS, lambda L, i, o: L.vb200_shrinkv(i, o, 3, 0), lambda a: orc.shrinkv(a, 3), in_place=True),
    Op("shrinkh", FORMATS, lambda L, i, o: L.vb200_shrinkh(i, o, 3, 0), lambda a: orc.shrinkh(a, 3)),
    Op("reducev", FORMATS, lambda L, i, o: L.vb200_reducev(i, o, 1.7, LANCZOS3, 0.0),
       lambda a: orc.reducev(a, 1.7, "lanczos3", 0.0, rect_h=16)),
    Op("reduceh", FORMATS, lambda L, i, o: L.vb200_reduceh(i, o, 1.7, LANCZOS3, 0.0),
       lambda a: orc.reduceh(a, 1.7, "lanczos3", 0.0, rect_w=0)),
    Op("reduce", FORMATS, lambda L, i, o: L.vb200_reduce(i, o, 2.3, 1.7, LANCZOS3, 0.0),
       lambda a: orc.reduceh(orc.reducev(a, 1.7, "lanczos3", 0.0, rect_h=16), 2.3, "lanczos3", 0.0, rect_w=0)),
    Op("resize_down", FORMATS, lambda L, i, o: L.vb200_resize(i, o, 0.6, 0.6, LANCZOS3, 2.0), lambda a: orc.resize(a, 0.6)),
    Op("resize_up", FORMATS, lambda L, i, o: L.vb200_resize(i, o, 1.7, 1.7, LANCZOS3, 2.0), lambda a: orc.resize(a, 1.7)),
    Op("premultiply", FORMATS, lambda L, i, o: L.vb200_premultiply(i, o, 255.0, 0), lambda a: orc.premultiply(a, 255.0, False)),
    Op("unpremultiply", FORMATS, lambda L, i, o: L.vb200_unpremultiply(i, o, 255.0, 0),
       lambda a: orc.unpremultiply(a, 255.0, False)),
    Op("premultiply_uchar", U8, lambda L, i, o: L.vb200_premultiply(i, o, 255.0, 1), lambda a: orc.premultiply(a, 255.0, True),
       bands=(2, 3, 4), in_place=True),
    Op("unpremultiply_uchar", U8, lambda L, i, o: L.vb200_unpremultiply(i, o, 255.0, 1),
       lambda a: orc.unpremultiply(a, 255.0, True), bands=(2, 3, 4), in_place=True),
    Op("conv", FORMATS, _mask_call("vb200_conv", M33, 1.3, 0.5, vb.PRECISIONS["float"]),
       lambda a: pyconv.conv(a, M33, 1.3, 0.5, "float")),
    Op("conv_integer", FORMATS, _mask_call("vb200_conv", MI33, 7.0, 1.0, vb.PRECISIONS["integer"]),
       lambda a: pyconv.conv(a, MI33, 7.0, 1.0, "integer"), in_place=True),
    Op("convsep", FORMATS, _mask_call("vb200_convsep", SEP5, 16.0, 0.0, vb.PRECISIONS["integer"]),
       lambda a: pyconv.convsep(a, SEP5, 16.0, 0.0, "integer")),
    Op("gaussblur", FORMATS, lambda L, i, o: L.vb200_gaussblur(i, o, 1.0, 0.2, vb.PRECISIONS["float"]),
       lambda a: pyconv.gaussblur(a, 1.0, 0.2, "float")),
    Op("sharpen", U8, lambda L, i, o: L.vb200_sharpen(i, o, 0.5, 2.0, 10.0, 20.0, 0.0, 3.0), lambda a: pyconv.sharpen(a, "srgb"),
       in_place=True),
    Op("flatten", FORMATS, _flatten_call, lambda a: pyconv.flatten(a, FLATTEN_BG, flatten_max_alpha(a.dtype)),
       bands=(4,)),
    Op("morph", U8, _mask_call("vb200_morph", CROSS, 1.0, 0.0, 0), lambda a: pyconv.morph(a, CROSS, "erode"), bands=(1, 3, 4),
       in_place=True),
    Op("rank", FORMATS, lambda L, i, o: L.vb200_rank(i, o, 3, 3, 2), lambda a: pyconv.rank(a, 3, 3, 2), in_place=True),
    Op("median", FORMATS, lambda L, i, o: L.vb200_median(i, o, 3), lambda a: pyconv.median(a, 3), in_place=True),
    _colour_op("srgb", "lab", np.uint8, (3, 4)),
    _colour_op("lab", "srgb", np.float32, (3,)),
    _colour_op("xyz", "lab", np.float32, (3, 4)),
    _colour_op("rgb16", "srgb", np.uint16, (3,)),
    _colour_op("labs", "lab", np.int16, (3,)),
    _colour_op("b-w", "srgb", np.uint8, (1,)),
    _colour_op("srgb", "b-w", np.uint8, (3, 4)),
] + _icc_ops()
OP = {op.name: op for op in OPS}
# the ops whose in-place form is asked for: the result has the input's format and fits in it
IN_PLACE = [op.name for op in OPS if op.in_place]


def inputs(op, seed):
    """(array, interpretation, layout) for every format, band count, shape and layout of an op"""
    rng = np.random.default_rng(seed)
    for dt in op.formats:
        for b in op.bands:
            for h, w in SHAPES:
                a = op.make(rng, dt, (h, w, b))
                for layout in layouts(dt, b):
                    yield a, op.interp_for(b), layout


def run(op, cin, cout):
    vb._check(op.call(vb.lib(), C.byref(cin), C.byref(cout)))


# ------------------------------------------------------------------------------------------------ the vector kernels

def _aligned(off, bpl, grid):
    return off % grid == 0 and bpl % grid == 0


# kernel -> the layout half of its dispatch condition (input at (off, bpl); library-allocated outputs are on every grid),
# plus the rest of the condition given the image: (dtype, w, bands, extra)
VECTOR_PATHS = {
    # resample_kernels.cu dev_shrinkv: (ne & 3) == 0 && aligned4(in) && aligned4(out) && vshrink <= 257
    "shrinkv_u8x4": lambda off, bpl, dt, w, b, x: dt == np.uint8 and (w * b) % 4 == 0 and _aligned(off, bpl, 4) and x <= 257,
    # run_reducev: (ne & 3) == 0 && aligned4(in) && aligned4(out) (staged when also on the 16-byte grid with ne % 16 == 0)
    "reducev_u8_dp2a": lambda off, bpl, dt, w, b, x: dt == np.uint8 and (w * b) % 4 == 0 and _aligned(off, bpl, 4),
    # run_reduceh: bands == 4 && aligned4(in) && aligned4(out)
    "reduceh_u8x4_dp2a": lambda off, bpl, dt, w, b, x: dt == np.uint8 and b == 4 and _aligned(off, bpl, 4),
    # premul_u8_kernel's word path: bands == 4 && aligned4(in) && aligned4(out)
    "premul_u8_words": lambda off, bpl, dt, w, b, x: dt == np.uint8 and b == 4 and _aligned(off, bpl, 4),
    # flatten_can_x4: uchar, 4 bands, w % 4 == 0, in on the 16-byte grid, out on the 4-byte grid
    "flatten_u8x4": lambda off, bpl, dt, w, b, x: dt == np.uint8 and b == 4 and w % 4 == 0 and _aligned(off, bpl, 16),
    # colour.cu dev_colourspace: 3 bands, w % 4 == 0, in and out on the 16-byte grid (sRGB <-> Lab)
    "colour_x4": lambda off, bpl, dt, w, b, x: b == 3 and w % 4 == 0 and _aligned(off, bpl, 16),
    # affine.cu dev_affine_scale: uchar, 4 bands, bicubic, in on the 4-byte grid (separable unless VB200_NO_AFFINE_SEP)
    "affine_bicubic_u8x4": lambda off, bpl, dt, w, b, x: dt == np.uint8 and b == 4 and _aligned(off, bpl, 4),
    # sharpen_fused.cu dev_sharpen_fused: 3 bands always, 4 bands only with base and strides on the 4-byte grid
    "sharpen_fused": lambda off, bpl, dt, w, b, x: b == 3 or _aligned(off, bpl, 4),
}


def _vector_cases():
    """(kernel, op name, dtype, (h, w, bands), layout, extra, env): each vector kernel on both sides of its condition"""
    out = []
    for layout in ("packed", "padded", "word", "byte1", "byte3"):
        out += [("shrinkv_u8x4", "shrinkv", np.uint8, (24, 256, 4), layout, 3, None),
                ("reducev_u8_dp2a", "reducev", np.uint8, (24, 256, 4), layout, 0, None),
                ("reduceh_u8x4_dp2a", "reduceh", np.uint8, (24, 256, 4), layout, 0, None),
                ("premul_u8_words", "premultiply_uchar", np.uint8, (24, 256, 4), layout, 0, None),
                ("premul_u8_words", "unpremultiply_uchar", np.uint8, (24, 256, 4), layout, 0, None),
                ("flatten_u8x4", "flatten", np.uint8, (24, 256, 4), layout, 0, None),
                ("colour_x4", "colour_srgb_lab", np.uint8, (24, 256, 3), layout, 0, None),
                ("affine_bicubic_u8x4", "resize_up", np.uint8, (24, 64, 4), layout, 0, None),
                ("affine_bicubic_u8x4", "resize_up", np.uint8, (24, 64, 4), layout, 0, "VB200_NO_AFFINE_SEP"),
                ("sharpen_fused", "sharpen", np.uint8, (40, 64, 4), layout, 0, None),
                ("sharpen_fused", "sharpen", np.uint8, (40, 64, 3), layout, 0, None)]
    for layout in ("packed", "offset", "padded"):
        out.append(("colour_x4", "colour_lab_srgb", np.float32, (24, 256, 3), layout, 0, None))
    # the rest of each condition, on the packed layout
    out += [("shrinkv_u8x4", "shrinkv257", np.uint8, (520, 64, 4), "packed", 257, None),
            ("shrinkv_u8x4", "shrinkv258", np.uint8, (520, 64, 4), "packed", 258, None),
            ("shrinkv_u8x4", "shrinkv", np.uint8, (24, 37, 3), "packed", 3, None),       # ne = 111: ne & 3 != 0
            ("reducev_u8_dp2a", "reducev", np.uint8, (24, 37, 3), "packed", 0, None),
            ("reduceh_u8x4_dp2a", "reduceh", np.uint8, (24, 256, 3), "packed", 0, None),
            ("premul_u8_words", "premultiply_uchar", np.uint8, (24, 37, 3), "packed", 0, None),
            ("flatten_u8x4", "flatten", np.uint8, (24, 255, 4), "packed", 0, None),       # w % 4 != 0
            ("colour_x4", "colour_srgb_lab", np.uint8, (24, 255, 3), "packed", 0, None),  # w % 4 != 0
            ("colour_x4", "colour_srgb_lab", np.uint8, (24, 256, 4), "packed", 0, None)]  # 4 bands
    return out


VECTOR_CASES = _vector_cases()
SHRINK_OPS = {"shrinkv257": 257, "shrinkv258": 258}


def vector_side(kernel, dt, shape, layout, extra):
    h, w, b = shape
    off, bpl = placement(layout, dt, w, b)
    return bool(VECTOR_PATHS[kernel](off, bpl, np.dtype(dt), w, b, extra))


# ------------------------------------------------------------------------------------------------ CPU

def test_layouts_leave_the_grids_they_claim():
    """padded and offset rows leave the 4-byte grid (uchar) or the 16-byte grid (wider types) yet stay on the element
    grid; word sits on the 4-byte grid only; byteN leaves every grid"""
    for dt in FORMATS:
        es = np.dtype(dt).itemsize
        for b in (1, 3, 4):
            for w in (37, 5, 256):
                line = w * b * es
                for layout in layouts(dt, b):
                    off, bpl = placement(layout, dt, w, b)
                    assert bpl >= line and off % es == 0 and bpl % es == 0, (dt, layout)
                    if layout in ("padded", "offset"):
                        assert (bpl - line) % (4 if es == 1 else 16) != 0, (dt, layout)
                    if layout == "word":
                        assert _aligned(off, bpl, 4) == (line % 4 == 0) and not _aligned(off, bpl, 16)
                    if layout.startswith("byte"):
                        assert off % 4 != 0 and bpl == line + 1
    assert layouts(np.uint8, 4)[-3:] == ["byte1", "byte2", "byte3"] and "byte1" not in layouts(np.uint16, 4)


def test_every_vector_kernel_is_reached_on_both_sides():
    sides = {}
    for kernel, name, dt, shape, layout, extra, env in VECTOR_CASES:
        sides.setdefault(kernel, set()).add(vector_side(kernel, dt, shape, layout, extra))
    assert set(sides) == set(VECTOR_PATHS)
    assert all(s == {True, False} for s in sides.values()), sides
    # the non-layout halves: vshrink 257 / 258, ne & 3, w % 4 and the band count each flip a packed case
    assert vector_side("shrinkv_u8x4", np.uint8, (520, 64, 4), "packed", 257)
    assert not vector_side("shrinkv_u8x4", np.uint8, (520, 64, 4), "packed", 258)
    assert not vector_side("shrinkv_u8x4", np.uint8, (24, 37, 3), "packed", 3)
    assert not vector_side("flatten_u8x4", np.uint8, (24, 255, 4), "packed", 0)
    assert not vector_side("colour_x4", np.uint8, (24, 255, 3), "packed", 0)
    assert vector_side("sharpen_fused", np.uint8, (40, 64, 4), "word", 0)
    assert not vector_side("sharpen_fused", np.uint8, (40, 64, 4), "byte1", 0)


def test_ops_cover_the_formats_they_take():
    """seven formats for resample, premultiply, conv, rank and flatten; uchar for morph and sharpen; uchar, ushort and
    float for ICC"""
    for name in ("shrinkv", "shrinkh", "reducev", "reduceh", "reduce", "resize_down", "resize_up", "premultiply",
                 "unpremultiply", "conv", "conv_integer", "convsep", "gaussblur", "flatten", "rank", "median"):
        assert OP[name].formats == FORMATS, name
    assert OP["morph"].formats == OP["sharpen"].formats == U8
    icc = {np.dtype(dt) for op in OPS if op.name.startswith("icc") for dt in op.formats}
    assert icc == {np.dtype(np.uint8), np.dtype(np.uint16), np.dtype(np.float32)}
    assert set(IN_PLACE) >= {"morph", "rank", "median", "shrinkv", "premultiply_uchar", "conv_integer", "sharpen"}


# ------------------------------------------------------------------------------------------------ GPU: every layout

@pytest.mark.gpu
@pytest.mark.parametrize("name", [op.name for op in OPS])
def test_gpu_every_format_and_layout(vb, name):
    """a device input in every layout, library-allocated device output: the oracle's pixels, the descriptor filled in"""
    op = OP[name]
    for a, interp, layout in inputs(op, zlib.crc32(name.encode())):
        what = (name, a.dtype, a.shape, layout)
        cin, buf = device_image(a, layout, interp)
        cout = vb.CImage()
        run(op, cin, cout)
        shape, dt = op.expect(a)
        assert (cout.Ysize, cout.Xsize, cout.Bands) == shape and cout.BandFmt == fmt_of(dt), what
        assert cout.Type == (op.out_type if op.out_type is not None else interp), what
        op.check(take_device(cout), a, what)
        buf.assert_outside_untouched(what)


# ------------------------------------------------------------------------------------------------ GPU: output modes

def _out_layouts(es_out):
    """(base offset, extra pitch bytes) of a caller's output buffer: on the result's element grid, and off it"""
    return ((0, es_out), (1, 1)) if es_out > 1 else ((0, 3), (1, 1))


@pytest.mark.gpu
@pytest.mark.parametrize("name", [op.name for op in OPS])
def test_gpu_output_modes(vb, name):
    """library-allocated device output, a caller's device buffer and a caller's host buffer with padded pitches: the
    same pixels, nothing written outside the rows, the descriptor filled in with the caller's pointer and pitch"""
    op = OP[name]
    rng = np.random.default_rng(len(name))
    dt = op.formats[-1]
    b = op.bands[-1]
    interp = op.interp_for(b)
    a = op.make(rng, dt, (29, 37, b))
    shape, odt = op.expect(a)
    oh, ow, ob = shape
    es = np.dtype(odt).itemsize
    line = ow * ob * es
    out_type = op.out_type if op.out_type is not None else interp
    layout = "offset"

    cin, src = device_image(a, layout, interp)
    cout = vb.CImage()
    run(op, cin, cout)
    ref = take_device(cout)
    op.check(ref, a, (name, "allocated"))

    for host in (False, True):
        for off, pad in _out_layouts(es):
            what = (name, "host" if host else "device", off, pad)
            if host:
                hoff, hbpl = placement("padded", dt, a.shape[1], b)
                hin = Buf(a.shape[0], a.shape[1] * b * a.itemsize, hoff, hbpl, a, host=True)
                cin = vb.CImage(a.shape[1], a.shape[0], b, fmt_of(dt), interp, vb.HOST, C.c_void_p(hin.ptr), hbpl)
            dst = Buf(oh, line, off, line + pad, host=host)
            cout = vb.CImage(0, 0, 0, 0, 0, vb.HOST if host else vb.DEVICE, C.c_void_p(dst.ptr), line + pad)
            run(op, cin, cout)
            assert cout.data == dst.ptr and cout.bpl == line + pad, what
            assert (cout.Xsize, cout.Ysize, cout.Bands, cout.BandFmt, cout.Type) == (ow, oh, ob, fmt_of(odt), out_type), what
            assert cout.where == (vb.HOST if host else vb.DEVICE), what
            same(dst.rows(odt, ow, ob), ref, what)
            dst.assert_outside_untouched(what)
            if host:
                hin.assert_outside_untouched(what)
    src.assert_outside_untouched(name)


# ------------------------------------------------------------------------------------------------ GPU: in place

@pytest.mark.gpu
@pytest.mark.parametrize("name", IN_PLACE)
def test_gpu_in_place(vb, name):
    """out->data == in->data with the same bpl: the out-of-place result, the pitch padding untouched"""
    op = OP[name]
    rng = np.random.default_rng(7 + len(name))
    for b in op.bands:
        for layout in ("packed", "offset", "byte1" if b in (3, 4) else "word"):
            a = op.make(rng, np.uint8, (29, 37, b))
            interp = op.interp_for(b)
            want = op.want(a)
            cin, buf = device_image(a, layout, interp)
            cout = vb.CImage()
            run(op, cin, cout)
            out_of_place = take_device(cout)
            same(out_of_place, want, (name, layout, "out of place"))
            cout = vb.CImage(0, 0, 0, 0, 0, vb.DEVICE, cin.data, cin.bpl)
            run(op, cin, cout)
            what = (name, b, layout)
            assert cout.data == cin.data and cout.bpl == cin.bpl, what
            # the result's rows at the input's pitch (shrinkv: the first oh of them)
            same(buf.rows(np.uint8, a.shape[1], b)[:want.shape[0]], out_of_place, what)
            buf.assert_outside_untouched(what)


# ------------------------------------------------------------------------------------------------ GPU: pass-through steps

@pytest.mark.gpu
def test_gpu_pass_through_steps_return_a_separate_buffer(vb):
    """shrink by 1 and premultiply of a one-band image return their input: on the device with out->data = NULL the result
    is a buffer of its own with the same pixels, and freeing it leaves the input readable"""
    L = vb.lib()
    rng = np.random.default_rng(3)
    steps = [(lambda i, o: L.vb200_shrinkv(i, o, 1, 0), 3), (lambda i, o: L.vb200_shrinkh(i, o, 1, 0), 3),
             (lambda i, o: L.vb200_premultiply(i, o, 255.0, 0), 1), (lambda i, o: L.vb200_premultiply(i, o, 255.0, 1), 1),
             (lambda i, o: L.vb200_unpremultiply(i, o, 255.0, 0), 1)]
    for k, (step, b) in enumerate(steps):
        for dt in (np.uint8, np.int16, np.float32):
            a = pixels(rng, dt, (29, 37, b))
            cin, buf = device_image(a, "offset", SRGB if b == 3 else B_W)
            cout = vb.CImage()
            vb._check(step(C.byref(cin), C.byref(cout)))
            assert cout.data and cout.data != cin.data, (k, dt)
            same(take_device(cout), a, (k, dt))  # frees it
            same(buf.rows(a.dtype, 37, b), a, (k, dt, "input after the free"))
            cout = vb.CImage()
            vb._check(L.vb200_shrinkh(C.byref(cin), C.byref(cout), 2, 0))
            same(take_device(cout), orc.shrinkh(a, 2), (k, dt, "input still usable"))


# ------------------------------------------------------------------------------------------------ GPU: vector kernels

@pytest.mark.gpu
@pytest.mark.parametrize("case", VECTOR_CASES, ids=["%s-%s-%s-%dx%dx%d-%s%s" % (c[0], c[1], np.dtype(c[2]).name, *c[3], c[4],
                                                                                 "-nosep" if c[6] else "") for c in VECTOR_CASES])
def test_gpu_vector_kernels_on_both_sides(vb, monkeypatch, case):
    """each vector kernel's case against the oracle; the 4-band sharpen also by its launch count (one fused kernel, or
    the unfused chain)"""
    kernel, name, dt, shape, layout, extra, env = case
    if env:
        monkeypatch.setenv(env, "1")
    rng = np.random.default_rng(zlib.crc32(("%s %s" % case[:2]).encode()))
    if name in SHRINK_OPS:
        f = SHRINK_OPS[name]
        op = Op(name, U8, lambda L_, i, o: L_.vb200_shrinkv(i, o, f, 0), lambda a: orc.shrinkv(a, f))
        a = pixels(rng, dt, shape)
        a[:, : shape[1] // 2] = 255  # every 16-bit lane at its largest sum
    else:
        op = OP[name]
        a = op.make(rng, dt, shape)
    cin, buf = device_image(a, layout, op.interp_for(shape[2]))
    cout = vb.CImage()
    n0 = vb.launch_count()
    run(op, cin, cout)
    launches = vb.launch_count() - n0
    op.check(take_device(cout), a, case)
    buf.assert_outside_untouched(case)
    if kernel == "sharpen_fused":
        fused = vector_side(kernel, dt, shape, layout, extra)
        assert (launches == 1) == fused, (case, launches)


# ------------------------------------------------------------------------------------------------ GPU: refusals

@pytest.mark.gpu
def test_gpu_refusals_write_nothing(vb):
    """a stride shorter than a line (device or host), a device base or stride off the element grid, a padded device
    image to vb200_thumbnail_image, a device image to vb200_chain_run_host: -1 with a message and *out untouched; the
    next good call on the thread succeeds"""
    L = vb.lib()
    rng = np.random.default_rng(5)

    def refused(call, cin, match, what):
        dst = Buf(29, 64, 0, 64)
        for cout in (vb.CImage(), vb.CImage(0, 0, 0, 0, 0, vb.DEVICE, C.c_void_p(dst.ptr), 64)):
            before = bytes(cout)
            L.vb200_error_clear()
            assert call(C.byref(cin), C.byref(cout)) == -1, what
            msg = L.vb200_error_buffer().decode()
            L.vb200_error_clear()
            assert match in msg, (what, msg)
            assert bytes(cout) == before, (what, "descriptor written")
        assert (dst.bytes() == SENTINEL).all(), (what, "wrote into the caller's buffer")

    def good(a, interp=SRGB):
        cin, buf = device_image(a, "offset", interp)
        cout = vb.CImage()
        vb._check(L.vb200_shrinkh(C.byref(cin), C.byref(cout), 2, 0))
        same(take_device(cout), orc.shrinkh(a, 2), "good call after a refusal")

    calls = {"shrinkv": lambda i, o: L.vb200_shrinkv(i, o, 2, 0), "resize": lambda i, o: L.vb200_resize(i, o, 0.5, 0.5, 5, 2.0),
             "conv": lambda i, o: OP["conv"].call(L, i, o), "colourspace": lambda i, o: L.vb200_colourspace(i, o, LAB),
             "rank": lambda i, o: L.vb200_rank(i, o, 3, 3, 4), "flatten": lambda i, o: _flatten_call(L, i, o),
             "morph": lambda i, o: OP["morph"].call(L, i, o), "premultiply": lambda i, o: L.vb200_premultiply(i, o, 255.0, 1)}
    for dt in (np.uint8, np.uint16, np.float32):
        a = pixels(rng, dt, (29, 37, 3))
        es = a.itemsize
        line = 37 * 3 * es
        for cname, call in calls.items():
            if cname == "morph" and dt != np.uint8:
                continue
            buf = Buf(29, line, 0, line, a)
            short = vb.CImage(37, 29, 3, fmt_of(dt), SRGB, vb.DEVICE, C.c_void_p(buf.ptr), line - es)
            refused(call, short, "too small", (cname, dt, "device bpl < line"))
            host = np.ascontiguousarray(a)
            hshort = vb.CImage(37, 29, 3, fmt_of(dt), SRGB, vb.HOST, C.c_void_p(host.ctypes.data), line - 1)
            refused(call, hshort, "too small", (cname, dt, "host bpl < line"))
            if es > 1:
                for off, bpl in ((1, line + es), (0, line + 1), (es + 1, line + 2 * es + 1)):
                    b2 = Buf(29, line, off, bpl, a)
                    odd = vb.CImage(37, 29, 3, fmt_of(dt), SRGB, vb.DEVICE, C.c_void_p(b2.ptr), bpl)
                    refused(call, odd, "not a multiple", (cname, dt, off, bpl))
                    b2.assert_outside_untouched((cname, dt, off, bpl))
            good(a)

    # thumbnail_image: device frames must be packed
    a = rng.integers(0, 256, (64, 96, 4), dtype=np.uint8)
    thumb = lambda i, o: L.vb200_thumbnail_image(i, o, 32, 0, 0, 0)
    cin, buf = device_image(a, "padded", SRGB)
    refused(thumb, cin, "device frames must be packed", "thumbnail padded")
    cin, buf = device_image(a, "packed", SRGB)
    cout = vb.CImage()
    vb._check(thumb(C.byref(cin), C.byref(cout)))
    same(take_device(cout), orc.thumbnail_image(a, 32), "thumbnail packed device frame")

    # the chain pump takes host images only
    chain = vb.Chain().rank(3, 3, 4)
    cin, buf = device_image(a, "packed", SRGB)
    cins, couts = (vb.CImage * 1)(cin), (vb.CImage * 1)()
    L.vb200_error_clear()
    assert L.vb200_chain_run_host(chain._p, cins, couts, 1) == -1
    msg = L.vb200_error_buffer().decode()
    L.vb200_error_clear()
    assert "is not a host image" in msg, msg
    assert bytes(couts[0]) == bytes(vb.CImage())
    assert np.array_equal(chain.run([a])[0].numpy(), pyconv.rank(a, 3, 3, 4))
    chain.close()
    good(a[:29, :37, :3].copy())

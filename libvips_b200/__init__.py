"""libvips_b200 -- Python mirror of the libvips operator interface for the
H100-native pixel hot path, bound over the C ABI of libvb200.so (include/vb200.h).

The class and method names follow pyvips / the libvips C API
(vips_reducev, vips_resize, vips_thumbnail_image, vips_conv, vips_colourspace ...)
so tests read like the reference's own test-suite.  All pixels are produced by
CUDA kernels inside libvb200.so: there is no CPU fallback here, and importing
the operators without the built library (or calling them without a GPU) raises.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.environ.get("VB200_LIB") or os.path.join(_HERE, "libvb200.so")  # VB200_LIB: tuning builds (tools/build_variant.sh)
_lib = None

HOST, DEVICE = 0, 1

FORMATS = {np.dtype(np.uint8): 0, np.dtype(np.int8): 1, np.dtype(np.uint16): 2, np.dtype(np.int16): 3,
           np.dtype(np.uint32): 4, np.dtype(np.int32): 5, np.dtype(np.float32): 6, np.dtype(np.float64): 8}
DTYPES = {v: k for k, v in FORMATS.items()}
KERNELS = {"nearest": 0, "linear": 1, "cubic": 2, "mitchell": 3, "lanczos2": 4, "lanczos3": 5,
           "mks2013": 6, "mks2021": 7}
SIZES = {"both": 0, "up": 1, "down": 2, "force": 3}
PRECISIONS = {"integer": 0, "float": 1, "approximate": 2}
INTENTS = {"perceptual": 0, "relative": 1, "saturation": 2, "absolute": 3}
PCS = {"lab": 0, "xyz": 1}
INTERPRETATIONS = {"multiband": 0, "b-w": 1, "cmyk": 15, "xyz": 12, "lab": 13, "lch": 19, "labs": 21, "srgb": 22,
                   "yxy": 23, "rgb16": 25, "grey16": 26, "scrgb": 28, "hsv": 29}


class Error(Exception):
    """Raised with the text of vb200_error_buffer(), like pyvips.Error."""


class CImage(C.Structure):
    _fields_ = [("Xsize", C.c_int), ("Ysize", C.c_int), ("Bands", C.c_int), ("BandFmt", C.c_int),
                ("Type", C.c_int), ("where", C.c_int), ("data", C.c_void_p), ("bpl", C.c_size_t)]


class CRect(C.Structure):
    _fields_ = [("left", C.c_int), ("top", C.c_int), ("width", C.c_int), ("height", C.c_int)]


class CRegion(C.Structure):
    _fields_ = [("im", CImage), ("valid", CRect), ("data", C.c_void_p), ("bpl", C.c_int)]


class CMask(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("coeff", C.POINTER(C.c_double)), ("scale", C.c_double),
                ("offset", C.c_double)]


class CReduceParams(C.Structure):
    _fields_ = [("n_point", C.c_int), ("kernel", C.c_int), ("residual_shrink", C.c_double),
                ("offset", C.c_double)]


def library_path():
    return _LIB_PATH


def lib():
    """Load libvb200.so.  Fails loudly if the CUDA extension is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise Error("libvb200.so is not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                        "(there is no CPU fallback)")
        L = C.CDLL(_LIB_PATH)
        L.vb200_error_buffer.restype = C.c_char_p
        L.vb200_launch_count.restype = C.c_uint64
        L.vb200_get_stream.restype = C.c_void_p
        L.vb200_set_stream.argtypes = [C.c_void_p]
        L.vb200_format_sizeof.restype = C.c_size_t
        L.vb200_host_alloc.restype = C.c_void_p
        L.vb200_host_alloc.argtypes = [C.c_size_t]
        L.vb200_host_free.argtypes = [C.c_void_p]
        IP = C.POINTER(CImage)
        L.vb200_shrinkv.argtypes = [IP, IP, C.c_int, C.c_int]
        L.vb200_shrinkh.argtypes = [IP, IP, C.c_int, C.c_int]
        L.vb200_reducev.argtypes = [IP, IP, C.c_double, C.c_int, C.c_double]
        L.vb200_reduceh.argtypes = [IP, IP, C.c_double, C.c_int, C.c_double]
        L.vb200_reduce.argtypes = [IP, IP, C.c_double, C.c_double, C.c_int, C.c_double]
        L.vb200_resize.argtypes = [IP, IP, C.c_double, C.c_double, C.c_int, C.c_double]
        L.vb200_premultiply.argtypes = [IP, IP, C.c_double, C.c_int]
        L.vb200_unpremultiply.argtypes = [IP, IP, C.c_double, C.c_int]
        L.vb200_thumbnail_image.argtypes = [IP, IP, C.c_int, C.c_int, C.c_int, C.c_int]
        L.vb200_colourspace.argtypes = [IP, IP, C.c_int]
        MP = C.POINTER(CMask)
        L.vb200_conv.argtypes = [IP, IP, MP, C.c_int]
        L.vb200_convsep.argtypes = [IP, IP, MP, C.c_int]
        L.vb200_gaussblur.argtypes = [IP, IP, C.c_double, C.c_double, C.c_int]
        L.vb200_sharpen.argtypes = [IP, IP] + [C.c_double] * 6
        L.vb200_gaussmat.argtypes = [MP, C.c_double, C.c_double, C.c_int, C.c_int]
        L.vb200_mask_free.argtypes = [MP]
        L.vb200_image_free.argtypes = [IP]
        L.vb200_thumbnail_plan_new.restype = C.c_void_p
        L.vb200_thumbnail_plan_new.argtypes = [C.c_int] * 9
        PI = C.POINTER(C.c_int)
        L.vb200_jpeg_decode_batch.argtypes = [C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_int, C.c_int, C.c_void_p, C.c_int,
                                              C.c_size_t, C.c_size_t, PI, PI, PI]
        L.vb200_debug_jpeg_decode.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_size_t, PI, PI, PI]
        L.vb200_thumbnail_jpegshrink.argtypes = [C.c_int] * 5
        L.vb200_jpegsave_batch.argtypes = [C.c_void_p, C.c_int, C.c_size_t, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                           C.c_void_p, C.c_int, C.c_size_t, C.POINTER(C.c_size_t)]
        L.vb200_thumbnail_buffer.argtypes = [C.c_void_p, C.c_size_t, IP, C.c_int, C.c_int, C.c_int]
        L.vb200_thumbnail_plan_run_jpeg.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_int, C.c_int,
                                                    C.c_void_p, C.c_int, C.c_size_t]
        L.vb200_thumbnail_plan_free.argtypes = [C.c_void_p]
        L.vb200_thumbnail_plan_output.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.vb200_thumbnail_plan_bytes_per_frame.restype = C.c_size_t
        L.vb200_thumbnail_plan_bytes_per_frame.argtypes = [C.c_void_p]
        L.vb200_thumbnail_plan_is_fused.argtypes = [C.c_void_p]
        L.vb200_thumbnail_plan_kernel.restype = C.c_char_p
        L.vb200_thumbnail_plan_kernel.argtypes = [C.c_void_p]
        L.vb200_thumbnail_batch_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                                   C.c_int]
        L.vb200_thumbnail_batch_host.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                                 C.c_int]
        RP = C.POINTER(CRegion)
        L.vb200_reducev_gen.argtypes = [RP, RP, C.POINTER(CReduceParams)]
        L.vb200_reduceh_gen.argtypes = [RP, RP, C.POINTER(CReduceParams)]
        L.vb200_shrinkv_gen.argtypes = [RP, RP, C.c_int]
        L.vb200_shrinkh_gen.argtypes = [RP, RP, C.c_int]
        L.vb200_conv_gen.argtypes = [RP, RP, C.POINTER(CMask), C.c_int]
        L.vb200_icc_import.argtypes = [IP, IP, C.c_char_p, C.c_size_t, C.c_int, C.c_int]
        L.vb200_icc_export.argtypes = [IP, IP, C.c_char_p, C.c_size_t, C.c_int, C.c_int, C.c_int]
        L.vb200_icc_transform.argtypes = [IP, IP, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_int, C.c_int]
        L.vb200_debug_icc_eval.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_char_p, C.c_size_t,
                                           C.c_char_p, C.c_size_t, C.c_int, C.c_int, C.c_int]
        L.vb200_colour_gen.argtypes = [RP, RP, C.c_int]
        L.vb200_sharpen_batch_device.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t] + [C.c_int] * 4 + [C.c_double] * 6
        L.vb200_thumbnail_plan_set_sharpen.argtypes = [C.c_void_p] + [C.c_double] * 6
        L.vb200_device_numa_node.restype = C.c_int
        L.vb200_morph.argtypes = [IP, IP, MP, C.c_int]
        L.vb200_chain_add_morph.argtypes = [C.c_void_p, MP, C.c_int]
        L.vb200_rank.argtypes = [IP, IP, C.c_int, C.c_int, C.c_int]
        L.vb200_debug_hsv_host.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]
        L.vb200_flatten.argtypes = [IP, IP, C.c_void_p, C.c_int, C.c_double]
        L.vb200_chain_add_flatten.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_double]
        L.vb200_debug_flatten_host.argtypes = [C.c_void_p] + [C.c_int] * 5 + [C.c_void_p, C.c_int, C.c_double, C.c_int, C.c_void_p]
        L.vb200_median.argtypes = [IP, IP, C.c_int]
        L.vb200_chain_add_rank.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.vb200_debug_rank_host.argtypes = [C.c_void_p] + [C.c_int] * 7 + [C.c_void_p]
        L.vb200_chain_new.restype = C.c_void_p
        L.vb200_chain_free.argtypes = [C.c_void_p]
        L.vb200_chain_add_resize.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_int, C.c_double]
        L.vb200_chain_add_reduce.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_int, C.c_double]
        L.vb200_chain_add_colourspace.argtypes = [C.c_void_p, C.c_int]
        L.vb200_chain_add_conv.argtypes = [C.c_void_p, MP, C.c_int]
        L.vb200_chain_add_convsep.argtypes = [C.c_void_p, MP, C.c_int]
        L.vb200_chain_add_gaussblur.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_int]
        L.vb200_chain_add_sharpen.argtypes = [C.c_void_p] + [C.c_double] * 6
        L.vb200_chain_add_premultiply.argtypes = [C.c_void_p, C.c_double, C.c_int]
        L.vb200_chain_add_unpremultiply.argtypes = [C.c_void_p, C.c_double, C.c_int]
        L.vb200_chain_run_host.argtypes = [C.c_void_p, IP, IP, C.c_int]
        _lib = L
    return _lib


def _check(rc):
    if rc != 0:
        msg = lib().vb200_error_buffer().decode(errors="replace")
        lib().vb200_error_clear()
        raise Error(msg.strip() or "vb200 call failed")


def init(device=0):
    _check(lib().vb200_init(device))


def shutdown():
    lib().vb200_shutdown()


def launch_count():
    return int(lib().vb200_launch_count())


def set_stream(handle):
    lib().vb200_set_stream(C.c_void_p(handle))


def set_tile_geometry(tile_width=0, tile_height=0, fatstrip_height=0, thinstrip_height=0):
    lib().vb200_set_tile_geometry(tile_width, tile_height, fatstrip_height, thinstrip_height)


def set_vector_convi(on):
    lib().vb200_set_vector_convi(int(on))


def gaussmat(sigma, min_ampl, separable=False, precision="integer"):
    """vips_gaussmat: returns (coefficients, scale, offset)."""
    m = CMask()
    _check(lib().vb200_gaussmat(C.byref(m), float(sigma), float(min_ampl), int(separable), PRECISIONS[precision]))
    a = np.ctypeslib.as_array(m.coeff, shape=(m.height, m.width)).copy()
    scale, offset = m.scale, m.offset
    lib().vb200_mask_free(C.byref(m))
    return a, scale, offset


def _k(kernel):
    return KERNELS[kernel] if isinstance(kernel, str) else int(kernel)


def _interp(name):
    return INTERPRETATIONS[name] if isinstance(name, str) else int(name)


class Image:
    """A host image (numpy array, H x W x Bands) with libvips-style operators."""

    def __init__(self, array, interpretation=None):
        a = np.ascontiguousarray(array)
        if a.ndim == 2:
            a = a[:, :, None]
        if a.dtype not in FORMATS:
            raise Error("unsupported dtype %s" % a.dtype)
        self.array = a
        if interpretation is None:
            interpretation = "b-w" if a.shape[2] < 3 else "srgb"
        self.interpretation = _interp(interpretation)

    # pyvips-style constructors / accessors
    @staticmethod
    def new_from_array(array, interpretation=None):
        return Image(array, interpretation)

    def numpy(self):
        return self.array

    @property
    def width(self):
        return self.array.shape[1]

    @property
    def height(self):
        return self.array.shape[0]

    @property
    def bands(self):
        return self.array.shape[2]

    @property
    def format(self):
        return self.array.dtype

    def avg(self):
        return float(self.array.mean())

    def _c(self):
        a = self.array
        return CImage(a.shape[1], a.shape[0], a.shape[2], FORMATS[a.dtype], self.interpretation, HOST,
                      C.c_void_p(a.ctypes.data), a.strides[0])

    def _call(self, fn, *args):
        cin = self._c()
        cout = CImage()
        _check(fn(C.byref(cin), C.byref(cout), *args))
        n = cout.Ysize * cout.bpl
        buf = (C.c_uint8 * n).from_address(cout.data)
        dt = DTYPES[cout.BandFmt]
        arr = np.frombuffer(buf, dtype=dt).reshape(cout.Ysize, cout.Xsize, cout.Bands).copy()
        lib().vb200_image_free(C.byref(cout))
        return Image(arr, cout.Type)

    # ---- resample
    def shrinkv(self, vshrink, ceil=False):
        return self._call(lib().vb200_shrinkv, int(vshrink), int(ceil))

    def shrinkh(self, hshrink, ceil=False):
        return self._call(lib().vb200_shrinkh, int(hshrink), int(ceil))

    def reducev(self, vshrink, kernel="lanczos3", gap=0.0):
        return self._call(lib().vb200_reducev, float(vshrink), _k(kernel), float(gap))

    def reduceh(self, hshrink, kernel="lanczos3", gap=0.0):
        return self._call(lib().vb200_reduceh, float(hshrink), _k(kernel), float(gap))

    def reduce(self, hshrink, vshrink, kernel="lanczos3", gap=0.0):
        return self._call(lib().vb200_reduce, float(hshrink), float(vshrink), _k(kernel), float(gap))

    def resize(self, scale, vscale=None, kernel="lanczos3", gap=2.0):
        return self._call(lib().vb200_resize, float(scale), float(scale if vscale is None else vscale),
                          _k(kernel), float(gap))

    def premultiply(self, max_alpha=0.0, uchar=False):
        return self._call(lib().vb200_premultiply, float(max_alpha), int(uchar))

    def unpremultiply(self, max_alpha=0.0, uchar=False):
        return self._call(lib().vb200_unpremultiply, float(max_alpha), int(uchar))

    def thumbnail_image(self, width, height=None, size="both", linear=False):
        return self._call(lib().vb200_thumbnail_image, int(width), int(height or 0), SIZES[size], int(linear))

    # ---- convolution
    @staticmethod
    def _mask(mask, scale, offset):
        m = np.ascontiguousarray(mask, np.float64)
        if m.ndim == 1:
            m = m[None, :]
        return m, CMask(m.shape[1], m.shape[0], m.ctypes.data_as(C.POINTER(C.c_double)), float(scale), float(offset))

    def conv(self, mask, scale=1.0, offset=0.0, precision="float"):
        m, cm = self._mask(mask, scale, offset)
        return self._call(lib().vb200_conv, C.byref(cm), PRECISIONS[precision])

    def convsep(self, mask, scale=1.0, offset=0.0, precision="float"):
        m, cm = self._mask(mask, scale, offset)
        return self._call(lib().vb200_convsep, C.byref(cm), PRECISIONS[precision])

    def gaussblur(self, sigma, min_ampl=0.2, precision="integer"):
        return self._call(lib().vb200_gaussblur, float(sigma), float(min_ampl), PRECISIONS[precision])

    def sharpen(self, sigma=0.5, x1=2.0, y2=10.0, y3=20.0, m1=0.0, m2=3.0):
        return self._call(lib().vb200_sharpen, float(sigma), float(x1), float(y2), float(y3), float(m1), float(m2))

    # ---- conversion
    def flatten(self, background=None, max_alpha=0.0):
        """vips_flatten: blend the alpha band out against `background` (1 or bands - 1 values; None: black)"""
        bg = np.ascontiguousarray([] if background is None else background, np.float64).ravel()
        return self._call(lib().vb200_flatten, bg.ctypes.data_as(C.c_void_p) if len(bg) else None, len(bg), float(max_alpha))

    # ---- morphology
    def morph(self, mask, morph):
        """vips_morph: mask elements 0 / 128 / 255; morph "erode" or "dilate" """
        m, cm = self._mask(mask, 1.0, 0.0)
        return self._call(lib().vb200_morph, C.byref(cm), {"erode": 0, "dilate": 1}.get(morph, morph))

    def erode(self, mask):
        return self.morph(mask, "erode")

    def dilate(self, mask):
        return self.morph(mask, "dilate")

    def rank(self, width, height, index):
        """vips_rank: the index-th smallest element of every width x height window"""
        return self._call(lib().vb200_rank, int(width), int(height), int(index))

    def median(self, size):
        return self._call(lib().vb200_median, int(size))

    # ---- colour
    def colourspace(self, space, source_space=None):
        src = self if source_space is None else Image(self.array, source_space)
        return src._call(lib().vb200_colourspace, _interp(space))

    # ---- ICC (profiles are bytes: what vips_profile_load hands on)
    def icc_import(self, profile, intent="relative", pcs="lab"):
        return self._call(lib().vb200_icc_import, profile, len(profile), INTENTS[intent], PCS[pcs])

    def icc_export(self, profile, intent="relative", depth=8, pcs="lab"):
        return self._call(lib().vb200_icc_export, profile, len(profile), INTENTS[intent], int(depth), PCS[pcs])

    def icc_transform(self, output_profile, input_profile, intent="relative", depth=8):
        return self._call(lib().vb200_icc_transform, input_profile, len(input_profile), output_profile, len(output_profile),
                          INTENTS[intent], int(depth))


class JpegBatch:
    """n JPEG streams (bytes objects) as the pointer / length arrays the C ABI takes; keeps them alive."""

    def __init__(self, streams):
        self.streams = [bytes(s) for s in streams]
        self.n = len(self.streams)
        self._bufs = [C.create_string_buffer(s, len(s)) for s in self.streams]
        self.ptrs = (C.c_void_p * self.n)(*[C.cast(b, C.c_void_p) for b in self._bufs])
        self.lens = (C.c_size_t * self.n)(*[len(s) for s in self.streams])
        self.nbytes = sum(len(s) for s in self.streams)


def jpeg_geometry(streams, shrink=1):
    """(width, height, bands) the streams decode to at `shrink` (they must agree); no GPU needed"""
    b = streams if isinstance(streams, JpegBatch) else JpegBatch(streams)
    w, h, bands = C.c_int(), C.c_int(), C.c_int()
    _check(lib().vb200_jpeg_decode_batch(b.ptrs, b.lens, b.n, int(shrink), None, HOST, 0, 0, C.byref(w), C.byref(h), C.byref(bands)))
    return w.value, h.value, bands.value


def jpeg_decode_batch(streams, shrink=1, out_ptr=None):
    """vips_jpegload_buffer(..., shrink=shrink) of every stream on the device -> uint8 [n, h, w, bands] (host),
    or into the device pointer out_ptr (packed frames)"""
    b = streams if isinstance(streams, JpegBatch) else JpegBatch(streams)
    w, h, bands = jpeg_geometry(b, shrink)
    ww, hh, bb = C.c_int(), C.c_int(), C.c_int()
    if out_ptr is not None:
        _check(lib().vb200_jpeg_decode_batch(b.ptrs, b.lens, b.n, int(shrink), C.c_void_p(out_ptr), DEVICE, w * bands, w * h * bands,
                                             C.byref(ww), C.byref(hh), C.byref(bb)))
        return w, h, bands
    out = np.empty((b.n, h, w, bands), np.uint8)
    _check(lib().vb200_jpeg_decode_batch(b.ptrs, b.lens, b.n, int(shrink), out.ctypes.data_as(C.c_void_p), HOST, w * bands,
                                         w * h * bands, C.byref(ww), C.byref(hh), C.byref(bb)))
    return out


def jpeg_decode_host_twin(stream, shrink=1):
    """the decoder's per-block code compiled for the host (vb200_debug_jpeg_decode): what the CPU tests pin to libjpeg-turbo"""
    stream = bytes(stream)
    w, h, bands = C.c_int(), C.c_int(), C.c_int()
    _check(lib().vb200_debug_jpeg_decode(stream, len(stream), int(shrink), None, 0, C.byref(w), C.byref(h), C.byref(bands)))
    out = np.empty((h.value, w.value, bands.value), np.uint8)
    _check(lib().vb200_debug_jpeg_decode(stream, len(stream), int(shrink), out.ctypes.data_as(C.c_void_p), w.value * bands.value,
                                         C.byref(w), C.byref(h), C.byref(bands)))
    return out


def rank_host_twin(a, width, height, index):
    """rank.cu's tile staging + radix select compiled for the host (vb200_debug_rank_host): what the CPU tests pin to rank.c"""
    a = np.ascontiguousarray(a)
    if a.ndim == 2:
        a = a[:, :, None]
    out = np.empty_like(a)
    _check(lib().vb200_debug_rank_host(a.ctypes.data_as(C.c_void_p), a.shape[1], a.shape[0], a.shape[2], FORMATS[a.dtype], int(width),
                                       int(height), int(index), out.ctypes.data_as(C.c_void_p)))
    return out


def hsv_host_twin(a, to_hsv):
    """colour_ext.cu's sRGB <-> HSV per-pixel code compiled for the host (vb200_debug_hsv_host); a: (n, 3) uint8"""
    a = np.ascontiguousarray(a, np.uint8).reshape(-1, 3)
    out = np.empty_like(a)
    _check(lib().vb200_debug_hsv_host(a.ctypes.data_as(C.c_void_p), a.shape[0], int(bool(to_hsv)), out.ctypes.data_as(C.c_void_p)))
    return out


def flatten_host_twin(a, background=None, max_alpha=0.0, interpretation=None, x4=False):
    """flatten.cu's per-pixel code compiled for the host (vb200_debug_flatten_host): what the CPU tests pin to flatten.c"""
    a = np.ascontiguousarray(a)
    if a.ndim == 2:
        a = a[:, :, None]
    if interpretation is None:
        interpretation = 1 if a.shape[2] < 3 else 22
    bg = np.ascontiguousarray([] if background is None else background, np.float64).ravel()
    out = np.empty((a.shape[0], a.shape[1], max(1, a.shape[2] - 1)), a.dtype)
    _check(lib().vb200_debug_flatten_host(a.ctypes.data_as(C.c_void_p), a.shape[1], a.shape[0], a.shape[2], FORMATS[a.dtype],
                                          _interp(interpretation), bg.ctypes.data_as(C.c_void_p) if len(bg) else None, len(bg),
                                          float(max_alpha), int(x4), out.ctypes.data_as(C.c_void_p)))
    return out


_SAVE_BUFFERS = {}


def jpegsave_batch(frames, Q=75, subsample_mode="auto", in_ptr=None, shape=None, stride=None):
    """vips_jpegsave_buffer() of every frame of a uint8 array [n, h, w, bands] (bands 1 or 3) on the device -> list of bytes.
    in_ptr / shape: frames already on the device (packed), shape = (n, h, w, bands)"""
    mode = {"auto": 0, "on": 1, "off": 2}[subsample_mode]
    if in_ptr is None:
        frames = np.ascontiguousarray(frames)
        if frames.ndim == 3:
            frames = frames[..., None]
        n, h, w, bands = frames.shape
        src, where = frames.ctypes.data_as(C.c_void_p), HOST
    else:
        n, h, w, bands = shape
        src, where = C.c_void_p(in_ptr), DEVICE
    stride = int(stride or (w * h * bands * 2 + 4096))
    out = _SAVE_BUFFERS.get((n, stride))
    if out is None:
        _SAVE_BUFFERS.clear()          # one staging array, reused: a fresh quarter gigabyte per call is all page faults
        out = _SAVE_BUFFERS[(n, stride)] = np.empty((n, stride), np.uint8)
    lens = (C.c_size_t * n)()
    _check(lib().vb200_jpegsave_batch(src, where, w * bands, w * h * bands, n, w, h, bands, int(Q), mode, out.ctypes.data_as(C.c_void_p), HOST,
                                      stride, lens))
    return [out[i, :lens[i]].tobytes() for i in range(n)]


def thumbnail_buffer(stream, width, height=None, size="both"):
    """vips_thumbnail_buffer() of a JPEG stream: shrink-on-load decode + thumbnail on the device -> uint8 array"""
    stream = bytes(stream)
    out = CImage()
    out.where = HOST
    _check(lib().vb200_thumbnail_buffer(stream, len(stream), C.byref(out), int(width), int(height or 0), SIZES[size]))
    n = out.Ysize * out.bpl
    a = np.frombuffer(C.string_at(out.data, n), np.uint8).reshape(out.Ysize, out.bpl)[:, :out.Xsize * out.Bands]
    a = a.reshape(out.Ysize, out.Xsize, out.Bands).copy()
    lib().vb200_image_free(C.byref(out))
    return a


def thumbnail_jpegshrink(width, height, target_width, target_height=None, size="both"):
    """vips_thumbnail_find_jpegshrink (thumbnail.c:489-517)"""
    return int(lib().vb200_thumbnail_jpegshrink(width, height, target_width, target_height or 0, SIZES[size]))


class ThumbnailPlan:
    """The batched tile pump (vb200_thumbnail_plan_* in include/vb200.h)."""

    def __init__(self, width, height, bands=4, target_width=512, target_height=None, size="both",
                 has_alpha=None, linear=False):
        if has_alpha is None:
            # vips_image_hasalpha for the interpretation Image() guesses: B_W below 3 bands, sRGB from 3
            has_alpha = bands == 2 or bands >= 4
        self.width, self.height, self.bands = width, height, bands
        self._p = lib().vb200_thumbnail_plan_new(width, height, bands, 0, int(has_alpha), target_width,
                                                 target_height or 0, SIZES[size], int(linear))
        if not self._p:
            _check(-1)
        ow, oh = C.c_int(), C.c_int()
        lib().vb200_thumbnail_plan_output(self._p, C.byref(ow), C.byref(oh))
        self.out_width, self.out_height = ow.value, oh.value
        self.in_frame_bytes = width * height * bands
        self.out_frame_bytes = self.out_width * self.out_height * bands
        self.bytes_per_frame = int(lib().vb200_thumbnail_plan_bytes_per_frame(self._p))
        self.fused = bool(lib().vb200_thumbnail_plan_is_fused(self._p))
        self.kernel = lib().vb200_thumbnail_plan_kernel(self._p).decode()

    def set_sharpen(self, sigma=0.5, x1=2.0, y2=10.0, y3=20.0, m1=0.0, m2=3.0):
        """vips_sharpen appended to every batch of this plan (sigma <= 0: off); BASELINE config 5"""
        _check(lib().vb200_thumbnail_plan_set_sharpen(self._p, float(sigma), float(x1), float(y2), float(y3), float(m1),
                                                      float(m2)))

    def close(self):
        if self._p:
            lib().vb200_thumbnail_plan_free(self._p)
            self._p = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def run_device(self, in_ptr, out_ptr, n_frames, in_stride=None, out_stride=None):
        """Device pointers (ints); queued on the stream set with set_stream()."""
        _check(lib().vb200_thumbnail_batch_device(self._p, C.c_void_p(in_ptr), in_stride or self.in_frame_bytes,
                                                  C.c_void_p(out_ptr), out_stride or self.out_frame_bytes,
                                                  n_frames))

    def run_host_ptr(self, in_ptr, out_ptr, n_frames):
        _check(lib().vb200_thumbnail_batch_host(self._p, C.c_void_p(in_ptr), self.in_frame_bytes,
                                                C.c_void_p(out_ptr), self.out_frame_bytes, n_frames))

    def run_jpeg(self, streams, shrink, out_ptr=None):
        """JPEG streams decoded at `shrink` on the device and thumbnailed by this plan (made for the decoded
        geometry): -> uint8 [n, OH, OW, bands] on the host, or into the device pointer out_ptr"""
        b = streams if isinstance(streams, JpegBatch) else JpegBatch(streams)
        if out_ptr is not None:
            _check(lib().vb200_thumbnail_plan_run_jpeg(self._p, b.ptrs, b.lens, b.n, int(shrink), C.c_void_p(out_ptr), DEVICE,
                                                       self.out_frame_bytes))
            return None
        out = np.empty((b.n, self.out_height, self.out_width, self.bands), np.uint8)
        _check(lib().vb200_thumbnail_plan_run_jpeg(self._p, b.ptrs, b.lens, b.n, int(shrink), out.ctypes.data_as(C.c_void_p), HOST,
                                                   self.out_frame_bytes))
        return out

    def run_host(self, frames):
        """frames: uint8 array [n, H, W, bands] in host memory -> [n, OH, OW, bands]."""
        frames = np.ascontiguousarray(frames)
        assert frames.dtype == np.uint8 and frames.shape[1:] == (self.height, self.width, self.bands)
        out = np.empty((frames.shape[0], self.out_height, self.out_width, self.bands), np.uint8)
        self.run_host_ptr(frames.ctypes.data, out.ctypes.data, frames.shape[0])
        return out


class Chain:
    """An unfused operation graph pumped over a batch of host images (vb200_chain_* in include/vb200.h):
    the methods mirror Image's; run() takes a list of arrays (sizes may differ) and returns Images."""

    def __init__(self):
        self._p = lib().vb200_chain_new()
        if not self._p:
            _check(-1)
        self._keep = []

    def close(self):
        if self._p:
            lib().vb200_chain_free(self._p)
            self._p = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def resize(self, scale, vscale=None, kernel="lanczos3", gap=2.0):
        _check(lib().vb200_chain_add_resize(self._p, float(scale), float(scale if vscale is None else vscale), _k(kernel), float(gap)))
        return self

    def reduce(self, hshrink, vshrink, kernel="lanczos3", gap=0.0):
        _check(lib().vb200_chain_add_reduce(self._p, float(hshrink), float(vshrink), _k(kernel), float(gap)))
        return self

    def colourspace(self, space):
        _check(lib().vb200_chain_add_colourspace(self._p, _interp(space)))
        return self

    def conv(self, mask, scale=1.0, offset=0.0, precision="float"):
        m, cm = Image._mask(mask, scale, offset)
        _check(lib().vb200_chain_add_conv(self._p, C.byref(cm), PRECISIONS[precision]))
        return self

    def convsep(self, mask, scale=1.0, offset=0.0, precision="float"):
        m, cm = Image._mask(mask, scale, offset)
        _check(lib().vb200_chain_add_convsep(self._p, C.byref(cm), PRECISIONS[precision]))
        return self

    def morph(self, mask, morph):
        m, cm = Image._mask(mask, 1.0, 0.0)
        _check(lib().vb200_chain_add_morph(self._p, C.byref(cm), {"erode": 0, "dilate": 1}.get(morph, morph)))
        return self

    def flatten(self, background=None, max_alpha=0.0):
        bg = np.ascontiguousarray([] if background is None else background, np.float64).ravel()
        _check(lib().vb200_chain_add_flatten(self._p, bg.ctypes.data_as(C.c_void_p) if len(bg) else None, len(bg), float(max_alpha)))
        return self

    def rank(self, width, height, index):
        _check(lib().vb200_chain_add_rank(self._p, int(width), int(height), int(index)))
        return self

    def gaussblur(self, sigma, min_ampl=0.2, precision="integer"):
        _check(lib().vb200_chain_add_gaussblur(self._p, float(sigma), float(min_ampl), PRECISIONS[precision]))
        return self

    def sharpen(self, sigma=0.5, x1=2.0, y2=10.0, y3=20.0, m1=0.0, m2=3.0):
        _check(lib().vb200_chain_add_sharpen(self._p, float(sigma), float(x1), float(y2), float(y3), float(m1), float(m2)))
        return self

    def premultiply(self, max_alpha=0.0, uchar=False):
        _check(lib().vb200_chain_add_premultiply(self._p, float(max_alpha), int(uchar)))
        return self

    def unpremultiply(self, max_alpha=0.0, uchar=False):
        _check(lib().vb200_chain_add_unpremultiply(self._p, float(max_alpha), int(uchar)))
        return self

    def run(self, images):
        ims = [im if isinstance(im, Image) else Image(im) for im in images]
        n = len(ims)
        cin = (CImage * n)(*[im._c() for im in ims])
        cout = (CImage * n)()
        _check(lib().vb200_chain_run_host(self._p, cin, cout, n))
        res = []
        for o in cout:
            buf = (C.c_uint8 * (o.Ysize * o.bpl)).from_address(o.data)
            arr = np.frombuffer(buf, dtype=DTYPES[o.BandFmt]).reshape(o.Ysize, o.Xsize, o.Bands).copy()
            lib().vb200_image_free(C.byref(o))
            res.append(Image(arr, o.Type))
        return res

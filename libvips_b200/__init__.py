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
INTERPRETATIONS = {"multiband": 0, "b-w": 1, "histogram": 10, "cmyk": 15, "xyz": 12, "lab": 13, "lch": 19, "labs": 21, "srgb": 22,
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


class CThumbnailIcc(C.Structure):
    _fields_ = [("input_profile", C.c_char_p), ("input_len", C.c_size_t), ("output_profile", C.c_char_p), ("output_len", C.c_size_t),
                ("builtin_rgb", C.c_char_p), ("builtin_rgb_len", C.c_size_t), ("builtin_grey", C.c_char_p),
                ("builtin_grey_len", C.c_size_t), ("intent", C.c_int)]


def _icc_struct(output_profile, input_profile, intent, builtin_profiles):
    b = builtin_profiles or {}
    blob = lambda p: (bytes(p), len(p)) if p is not None else (None, 0)
    i, o, r, g = blob(input_profile), blob(output_profile), blob(b.get("srgb")), blob(b.get("sgrey"))
    return CThumbnailIcc(i[0], i[1], o[0], o[1], r[0], r[1], g[0], g[1], INTENTS[intent] if isinstance(intent, str) else int(intent))


def thumbnail_icc(output_profile=None, input_profile=None, intent="relative", builtin_profiles=None):
    """The VB200ThumbnailIcc of vips_thumbnail's output_profile / input_profile / intent (profiles are bytes);
    builtin_profiles: {"srgb": bytes, "sgrey": bytes}, what vips_profile_load gives for those names.  None when
    colour management is off."""
    if output_profile is None:
        return None
    return _icc_struct(output_profile, input_profile, intent, builtin_profiles)


def linear_icc(output_profile=None, input_profile=None, intent="relative", builtin_profiles=None):
    """The VB200ThumbnailIcc of vips_thumbnail(linear=TRUE)'s output_profile / input_profile / intent: unlike thumbnail_icc it is
    never None, since in linear mode an embedded profile alone turns colour management on"""
    return _icc_struct(output_profile, input_profile, intent, builtin_profiles)


def _embedded_arrays(embedded, n):
    """per-frame embedded profiles (a list of bytes / None) as the pointer and length arrays the C ABI takes"""
    if embedded is None:
        return None, None, None
    assert len(embedded) == n
    keep = [C.create_string_buffer(bytes(e), len(e)) if e else None for e in embedded]
    ptrs = (C.c_void_p * n)(*[C.cast(k, C.c_void_p) if k is not None else None for k in keep])
    lens = (C.c_size_t * n)(*[len(e) if e else 0 for e in embedded])
    return keep, ptrs, lens


def _icc_blob(fn, stream, *opts):
    stream = bytes(stream)
    n = C.c_size_t()
    _check(fn(stream, len(stream), *opts, None, 0, C.byref(n)))
    if n.value == 0:
        return None
    out = C.create_string_buffer(n.value)
    _check(fn(stream, len(stream), *opts, out, n.value, C.byref(n)))
    return out.raw[:n.value]


def jpeg_icc_profile(stream):
    """vips_image_get_blob(VIPS_META_ICC_NAME) of a JPEG stream (its APP2 ICC_PROFILE chunks): bytes, or None; no GPU"""
    return _icc_blob(lib().vb200_jpeg_icc_profile, stream)


def webp_icc_profile(stream):
    """vips_image_get_blob(VIPS_META_ICC_NAME) of a WebP stream (its ICCP chunk): bytes, or None; no GPU"""
    return _icc_blob(lib().vb200_webp_icc_profile, stream)


def png_icc_profile(stream):
    """vips_image_get_blob(VIPS_META_ICC_NAME) of a PNG stream (its iCCP chunk, inflated): bytes, or None; no GPU"""
    return _icc_blob(lib().vb200_png_icc_profile, stream)


class JpegSaveOptions(C.Structure):
    """VB200JpegSaveOptions"""
    _fields_ = [("Q", C.c_int), ("subsample_mode", C.c_int), ("optimize_coding", C.c_int), ("restart_interval", C.c_int),
                ("interlace", C.c_int)]


class PngSaveOptions(C.Structure):
    """VB200PngSaveOptions"""
    _fields_ = [("compression", C.c_int), ("strategy", C.c_int), ("xres", C.c_double), ("filter", C.c_int), ("interlace", C.c_int),
                ("bitdepth", C.c_int)]


PNG_STRATEGIES = {"default": 0, "filtered": 1}
PNG_FILTERS = {"none": 0x08, "sub": 0x10, "up": 0x20, "avg": 0x40, "paeth": 0x80, "all": 0xF8}   # VipsForeignPngFilter


def _png_options(compression, strategy, xres, filter="none", interlace=False, bitdepth=8):
    return PngSaveOptions(int(compression), PNG_STRATEGIES.get(strategy, strategy), float(xres), int(PNG_FILTERS.get(filter, filter)),
                          int(bool(interlace)), int(bitdepth))


class DzOptions(C.Structure):
    """VB200DzOptions"""
    _fields_ = [("layout", C.c_int), ("tile_size", C.c_int), ("overlap", C.c_int), ("depth", C.c_int), ("region_shrink", C.c_int),
                ("skip_blanks", C.c_int), ("container", C.c_int), ("suffix", C.c_char_p), ("jpeg", JpegSaveOptions)]


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
        SO = C.POINTER(JpegSaveOptions)
        L.vb200_jpegsave_batch_opts.argtypes = [C.c_void_p, C.c_int, C.c_size_t, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, SO,
                                                C.c_void_p, C.c_int, C.c_size_t, C.POINTER(C.c_size_t)]
        L.vb200_debug_jpeg_encode_opts.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, SO, C.c_void_p, C.c_size_t,
                                                   C.POINTER(C.c_size_t)]
        L.vb200_debug_jpeg_optimal_table.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.vb200_debug_jpeg_prog_events.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, SO, C.POINTER(C.c_ulonglong)]
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
        TI = C.POINTER(CThumbnailIcc)
        L.vb200_thumbnail_plan_set_icc.argtypes = [C.c_void_p, TI]
        L.vb200_thumbnail_plan_output_bands.argtypes = [C.c_void_p]
        L.vb200_thumbnail_batch_device_icc.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int,
                                                       C.c_void_p, C.c_void_p]
        L.vb200_thumbnail_batch_host_icc.argtypes = L.vb200_thumbnail_batch_device_icc.argtypes
        L.vb200_thumbnail_image_icc.argtypes = [IP, IP, C.c_int, C.c_int, C.c_int, TI, C.c_char_p, C.c_size_t]
        L.vb200_thumbnail_buffer_icc.argtypes = [C.c_void_p, C.c_size_t, IP, C.c_int, C.c_int, C.c_int, TI]
        L.vb200_jpeg_icc_profile.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.vb200_debug_icc_select.argtypes = [TI, C.c_int, C.c_char_p, C.c_size_t, C.POINTER(C.c_int)]
        L.vb200_debug_icc_classify.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_int]
        L.vb200_thumbnail_plan_set_linear_icc.argtypes = [C.c_void_p, TI]
        L.vb200_thumbnail_image_linear_icc.argtypes = [IP, IP, C.c_int, C.c_int, C.c_int, TI, C.c_char_p, C.c_size_t]
        L.vb200_thumbnail_buffer_linear_icc.argtypes = [C.c_void_p, C.c_size_t, IP, C.c_int, C.c_int, C.c_int, TI]
        L.vb200_debug_icc_select_linear.argtypes = [TI, C.c_int, C.c_char_p, C.c_size_t, PI, PI, PI]
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
        L.vb200_hist_find.argtypes = [IP, IP, C.c_int]
        L.vb200_hist_equal.argtypes = [IP, IP, C.c_int]
        L.vb200_hist_local.argtypes = [IP, IP, C.c_int, C.c_int, C.c_int]
        L.vb200_chain_add_hist_find.argtypes = [C.c_void_p, C.c_int]
        L.vb200_chain_add_hist_equal.argtypes = [C.c_void_p, C.c_int]
        L.vb200_chain_add_hist_local.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.vb200_debug_hist_local_host.argtypes = [C.c_void_p] + [C.c_int] * 7 + [C.c_void_p]
        L.vb200_debug_hist_equal_lut_host.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
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
        DO, PP = C.POINTER(DzOptions), C.POINTER(C.c_void_p)
        L.vb200_dzsave.argtypes = [IP, DO, PP]
        L.vb200_debug_dzsave.argtypes = [IP, DO, PP]
        L.vb200_dzsave_png.argtypes = [IP, DO, C.POINTER(PngSaveOptions), PP]
        L.vb200_debug_dzsave_png.argtypes = [IP, DO, C.POINTER(PngSaveOptions), PP]
        L.vb200_dz_free.argtypes = [C.c_void_p]
        L.vb200_dz_levels.argtypes = [C.c_void_p]
        L.vb200_dz_level_geometry.argtypes = [C.c_void_p, C.c_int, PI, PI, PI, PI]
        L.vb200_dz_tiles.argtypes = [C.c_void_p]
        L.vb200_dz_tiles.restype = C.c_long
        L.vb200_dz_tile.argtypes = [C.c_void_p, C.c_long] + [PI] * 7 + [PP, C.POINTER(C.c_size_t)]
        L.vb200_dz_tile_name.argtypes = [C.c_void_p, C.c_long, C.c_char_p, C.c_char_p, C.c_size_t]
        L.vb200_dz_sidecar.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.vb200_dz_pyramid_level.argtypes = [IP, C.c_int, IP]
        L.vb200_debug_dz_pyramid_level.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
        L.vb200_debug_dz_set_budget.argtypes = [C.c_size_t]
        L.vb200_debug_dz_pool_used.restype = C.c_size_t
        L.vb200_debug_dz_times.argtypes = [C.POINTER(C.c_float)]
        L.vb200_png_decode_batch.argtypes = [C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_int, C.c_void_p, C.c_int, C.c_size_t, C.c_size_t,
                                             PI, PI, PI]
        L.vb200_pngload_buffer.argtypes = [C.c_void_p, C.c_size_t, IP]
        L.vb200_png_icc_profile.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.vb200_thumbnail_plan_run_png.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_int, C.c_void_p, C.c_int,
                                                   C.c_size_t]
        L.vb200_debug_png_decode.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, PI, PI, PI]
        L.vb200_debug_inflate.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.vb200_debug_png_set_budget.argtypes = [C.c_size_t]
        L.vb200_gif_geometry.argtypes = [C.c_void_p, C.c_size_t, PI, PI, PI, PI]
        L.vb200_gif_decode_batch.argtypes = [C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                             C.c_size_t, C.c_size_t, PI, PI, PI]
        L.vb200_gifload_buffer.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, IP]
        L.vb200_thumbnail_plan_run_gif.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_int, C.c_void_p, C.c_int,
                                                   C.c_size_t]
        L.vb200_debug_gif_decode.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_size_t, PI, PI, PI]
        L.vb200_debug_lzw.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_uint, C.c_int, C.c_void_p, C.POINTER(C.c_size_t)]
        L.vb200_tiff_geometry.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, PI, PI, PI, PI, PI]
        L.vb200_tiff_decode_batch.argtypes = [C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                              C.c_int, C.c_size_t, C.c_size_t, PI, PI, PI]
        L.vb200_tiffload_buffer.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, IP]
        L.vb200_tiff_icc_profile.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.vb200_thumbnail_plan_run_tiff.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_int, C.c_int, C.c_int,
                                                    C.c_int, C.c_void_p, C.c_int, C.c_size_t]
        L.vb200_thumbnail_tiff_level.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, PI, PI]
        L.vb200_debug_thumbnail_pyramid_level.argtypes = [C.c_int, C.c_int, C.c_int, PI, PI, C.c_int, PI, PI, C.c_int, C.c_int, C.c_int,
                                                          PI, PI]
        L.vb200_debug_tiff_decode.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_size_t, PI, PI, PI]
        L.vb200_debug_tiff_lzw.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.POINTER(C.c_size_t)]
        L.vb200_webp_geometry.argtypes = [C.c_void_p, C.c_size_t, PI, PI, PI]
        L.vb200_webp_decode_batch.argtypes = [C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_int, C.c_void_p, C.c_int, C.c_size_t,
                                              C.c_size_t, PI, PI, PI]
        L.vb200_webpload_buffer.argtypes = [C.c_void_p, C.c_size_t, IP]
        L.vb200_webp_icc_profile.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.vb200_debug_webp_decode.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, PI, PI, PI]
        L.vb200_debug_webp_tables.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
        L.vb200_debug_webp_times.argtypes = [C.POINTER(C.c_float)]
        L.vb200_webp_decode_batch_scaled.argtypes = [C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_int, C.c_double, C.c_void_p, C.c_int,
                                                     C.c_size_t, C.c_size_t, PI, PI, PI]
        L.vb200_webpload_buffer_scaled.argtypes = [C.c_void_p, C.c_size_t, C.c_double, IP]
        L.vb200_debug_webp_decode_scaled.argtypes = [C.c_void_p, C.c_size_t, C.c_double, C.c_void_p, C.c_size_t, PI, PI, PI]
        L.vb200_debug_webp_rescale.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_size_t]
        L.vb200_thumbnail_webp_scale.argtypes = [C.c_int] * 5 + [C.POINTER(C.c_double), PI, PI]
        L.vb200_thumbnail_webp_buffer.argtypes = [C.c_void_p, C.c_size_t, IP, C.c_int, C.c_int, C.c_int, TI, C.c_int]
        L.vb200_thumbnail_plan_run_webp.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_int, C.c_double, C.c_void_p,
                                                    C.c_int, C.c_size_t]
        L.vb200_thumbnail_plan_new_pages.restype = C.c_void_p
        L.vb200_thumbnail_plan_new_pages.argtypes = [C.c_int] * 10
        L.vb200_thumbnail_plan_page_height.argtypes = [C.c_void_p]
        L.vb200_thumbnail_image_pages.argtypes = [IP, C.c_int, IP, C.c_int, C.c_int, C.c_int, TI, C.c_char_p, C.c_size_t, C.c_int, PI]
        L.vb200_thumbnail_plan_run_gif_pages.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_int, C.c_int, C.c_int,
                                                         C.c_void_p, C.c_int, C.c_size_t]
        L.vb200_thumbnail_buffer_pages.argtypes = [C.c_void_p, C.c_size_t, IP, C.c_int, C.c_int, C.c_int, TI, C.c_int, C.c_int, C.c_int, PI]
        PD = C.POINTER(C.c_double)
        L.vb200_debug_thumbnail_pages_size.argtypes = [C.c_int] * 6 + [PD, PD, PI, PI, PI]
        L.vb200_debug_thumbnail_pages_kernel.argtypes = [C.c_int] * 8 + [C.c_char_p, C.c_int]
        PO = C.POINTER(PngSaveOptions)
        L.vb200_pngsave_batch.argtypes = [C.c_void_p, C.c_int, C.c_size_t, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, PO, C.c_char_p,
                                          C.c_size_t, C.c_void_p, C.c_int, C.c_size_t, C.POINTER(C.c_size_t)]
        L.vb200_pngsave_buffer.argtypes = [IP, PO, C.c_char_p, C.c_size_t, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
        L.vb200_debug_png_encode.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, PO, C.c_char_p, C.c_size_t, C.c_void_p,
                                             C.c_size_t, C.POINTER(C.c_size_t)]
        L.vb200_debug_deflate.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
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

    def __init__(self, array, interpretation=None, page_height=None):
        a = np.ascontiguousarray(array)
        if a.ndim == 2:
            a = a[:, :, None]
        if a.dtype not in FORMATS:
            raise Error("unsupported dtype %s" % a.dtype)
        self.array = a
        if interpretation is None:
            interpretation = "b-w" if a.shape[2] < 3 else "srgb"
        self.interpretation = _interp(interpretation)
        # libvips' "page-height": pages of this many rows stacked vertically (a page strip); None = one page
        self.page_height = page_height

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
        return Image._take(cout)

    @staticmethod
    def _take(cout):
        dt = np.dtype(DTYPES[cout.BandFmt])
        buf = (C.c_uint8 * (cout.Ysize * cout.bpl)).from_address(cout.data)
        rows = np.frombuffer(buf, np.uint8).reshape(cout.Ysize, cout.bpl)[:, :cout.Xsize * cout.Bands * dt.itemsize]
        arr = rows.copy().view(dt).reshape(cout.Ysize, cout.Xsize, cout.Bands)
        lib().vb200_image_free(C.byref(cout))
        return Image(arr, cout.Type)

    @staticmethod
    def _load_buffer(fn, stream, *opts):
        """fn(stream, len, *opts, &out) of a vb200_*load_buffer, delivered to host memory -> Image"""
        stream = bytes(stream)
        out = CImage()
        out.where = HOST
        _check(fn(stream, len(stream), *opts, C.byref(out)))
        return Image._take(out)

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

    def thumbnail_image(self, width, height=None, size="both", linear=False, output_profile=None, input_profile=None,
                        intent="relative", embedded_profile=None, builtin_profiles=None):
        """vips_thumbnail_image; with output_profile, colour-managed as vips_thumbnail does (embedded_profile: the image's
        ICC blob; builtin_profiles: {"srgb": bytes, "sgrey": bytes})"""
        icc = thumbnail_icc(output_profile, input_profile, intent, builtin_profiles)
        if icc is None or linear:
            if icc is not None:
                raise Error("linear thumbnails with an output profile are not supported on the device path")
            if self.page_height is not None:
                return self._thumbnail_pages(width, height, size, None, None, linear)
            return self._call(lib().vb200_thumbnail_image, int(width), int(height or 0), SIZES[size], int(linear))
        emb = bytes(embedded_profile) if embedded_profile else None
        if self.page_height is not None:
            return self._thumbnail_pages(width, height, size, icc, emb, False)
        return self._call(lib().vb200_thumbnail_image_icc, int(width), int(height or 0), SIZES[size], C.byref(icc), emb,
                          len(emb) if emb else 0)

    def thumbnail_image_linear(self, width, height=None, size="both", output_profile=None, input_profile=None, intent="relative",
                               embedded_profile=None, builtin_profiles=None):
        """vips_thumbnail_image(linear=TRUE) with colour management: an embedded profile alone turns it on; with no profiles
        at all, the bytes of thumbnail_image(linear=True)"""
        icc = linear_icc(output_profile, input_profile, intent, builtin_profiles)
        emb = bytes(embedded_profile) if embedded_profile else None
        if self.page_height is not None:
            return self._thumbnail_pages(width, height, size, icc, emb, True)
        return self._call(lib().vb200_thumbnail_image_linear_icc, int(width), int(height or 0), SIZES[size], C.byref(icc), emb,
                          len(emb) if emb else 0)

    def _thumbnail_pages(self, width, height, size, icc, emb, linear):
        """vb200_thumbnail_image_pages: the strip thumbnailed as vips_thumbnail does (thumbnail.c:825-839), its page height
        set on the result (None when the result is one page)"""
        cin, cout, oph = self._c(), CImage(), C.c_int()
        _check(lib().vb200_thumbnail_image_pages(C.byref(cin), int(self.page_height), C.byref(cout), int(width), int(height or 0),
                                                 SIZES[size], C.byref(icc) if icc is not None else None, emb, len(emb) if emb else 0,
                                                 int(linear), C.byref(oph)))
        out = Image._take(cout)
        out.page_height = oph.value if oph.value < out.height else None
        return out

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

    # ---- histograms
    def hist_find(self, band=-1):
        """vips_hist_find: the (mx + 1) x 1 uint32 histogram of every band (band=-1) or of one band, interpretation histogram"""
        return self._call(lib().vb200_hist_find, int(band))

    def hist_equal(self, band=-1):
        """vips_hist_equal: equalise through the image's own cumulative histogram (band >= 0: that band's, for every band)"""
        return self._call(lib().vb200_hist_equal, int(band))

    def hist_local(self, width, height, max_slope=0):
        """vips_hist_local: local equalisation over a width x height window; max_slope > 0 limits the contrast (CLAHE).  Any
        max_slope >= 0 runs hist_local.c's arithmetic as written (the reference's argument range stops at 100)"""
        return self._call(lib().vb200_hist_local, int(width), int(height), int(max_slope))

    # ---- savers
    def dzsave(self, basename=None, **options):
        """vips_dzsave: the Deep Zoom / Zoomify tile pyramid of this image -> DzPyramid (see dzsave())"""
        return dzsave(self, basename, **options)

    def dzsave_png(self, basename=None, **options):
        """vips_dzsave with suffix ".png": the tile pyramid of this image with PNG tiles -> DzPyramid (see dzsave_png())"""
        return dzsave_png(self, basename, **options)

    def pngsave_buffer(self, compression=6, strategy="default", xres=1.0, profile=None, filter="none", interlace=False, bitdepth=8):
        """vips_pngsave_buffer: this uchar image (1-4 bands) as a PNG stream (bytes), deflated on the device; filter, interlace
        and bitdepth as in pngsave_batch"""
        cin = self._c()
        opts = _png_options(compression, strategy, xres, filter, interlace, bitdepth)
        prof = bytes(profile) if profile else None
        p, n = C.c_void_p(), C.c_size_t()
        _check(lib().vb200_pngsave_buffer(C.byref(cin), C.byref(opts), prof, len(prof) if prof else 0, C.byref(p), C.byref(n)))
        try:
            return C.string_at(p.value, n.value)
        finally:
            C.CDLL(None).free(p)

    @staticmethod
    def tiffload_buffer(stream, page=0, n=1, subifd=-1):
        """vips_tiffload_buffer(stream, page=page, n=n, subifd=subifd): the strips or tiles decoded on the device -> Image (uint8,
        B_W below 3 bands, sRGB from 3), with page_height set when more than one page loaded"""
        img = Image._load_buffer(lib().vb200_tiffload_buffer, stream, int(page), int(n), int(subifd))
        page_h = tiff_geometry(stream, page, subifd)[1]
        img.page_height = page_h if img.height > page_h else None
        return img

    @staticmethod
    def webpload_buffer(stream, scale=1.0):
        """vips_webpload_buffer(stream, scale=scale) of a lossy, still, opaque WebP: the frame decoded on the device -> Image
        (uint8, 3 bands, sRGB); scale != 1 is libwebp's scaled decode to rint(w * scale) x rint(h * scale)"""
        if scale == 1.0:
            return Image._load_buffer(lib().vb200_webpload_buffer, stream)
        return Image._load_buffer(lib().vb200_webpload_buffer_scaled, stream, float(scale))

    # ---- colour
    @staticmethod
    def gifload_buffer(stream, page=0, n=1):
        """vips_gifload_buffer(stream, page=page, n=n): the pages decoded on the device (n = -1: every page from `page` on),
        stacked vertically as libvips does -> Image (uint8, 3 or 4 bands), with page_height the screen height when more than
        one page loaded (nsgifload.c:279-280)"""
        img = Image._load_buffer(lib().vb200_gifload_buffer, stream, int(page), int(n))
        screen_h = gif_geometry(stream)[1]
        img.page_height = screen_h if img.height > screen_h else None
        return img

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


class StreamBatch:
    """n compressed streams (bytes objects: JPEG, PNG or GIF) as the pointer / length arrays the C ABI takes; keeps them alive."""

    def __init__(self, streams):
        self.streams = [bytes(s) for s in streams]
        self.n = len(self.streams)
        self._bufs = [C.create_string_buffer(s, len(s)) for s in self.streams]
        self.ptrs = (C.c_void_p * self.n)(*[C.cast(b, C.c_void_p) for b in self._bufs])
        self.lens = (C.c_size_t * self.n)(*[len(s) for s in self.streams])
        self.nbytes = sum(len(s) for s in self.streams)


JpegBatch = StreamBatch


def _batch_geometry(fn, streams, *opts):
    """(width, height, bands) vb200_*_decode_batch(streams, *opts) reports without an output (the streams must agree); no GPU"""
    b = streams if isinstance(streams, StreamBatch) else StreamBatch(streams)
    w, h, bands = C.c_int(), C.c_int(), C.c_int()
    _check(fn(b.ptrs, b.lens, b.n, *opts, None, HOST, 0, 0, C.byref(w), C.byref(h), C.byref(bands)))
    return w.value, h.value, bands.value


def _decode_batch(fn, streams, opts, out_ptr, out_bpl=None, out_frame_stride=None):
    """vb200_*_decode_batch(streams, *opts) -> uint8 [n, h, w, bands] (host), or into the device pointer out_ptr (packed
    frames unless out_bpl / out_frame_stride say otherwise) -> (w, h, bands)"""
    b = streams if isinstance(streams, StreamBatch) else StreamBatch(streams)
    w, h, bands = _batch_geometry(fn, b, *opts)
    if out_ptr is not None:
        bpl = out_bpl or w * bands
        _check(fn(b.ptrs, b.lens, b.n, *opts, C.c_void_p(out_ptr), DEVICE, bpl, out_frame_stride or bpl * h, None, None, None))
        return w, h, bands
    out = np.empty((b.n, h, w, bands), np.uint8)
    _check(fn(b.ptrs, b.lens, b.n, *opts, out.ctypes.data_as(C.c_void_p), HOST, w * bands, w * h * bands, None, None, None))
    return out


def jpeg_geometry(streams, shrink=1):
    """(width, height, bands) the streams decode to at `shrink` (they must agree); no GPU needed"""
    return _batch_geometry(lib().vb200_jpeg_decode_batch, streams, int(shrink))


def jpeg_decode_batch(streams, shrink=1, out_ptr=None):
    """vips_jpegload_buffer(..., shrink=shrink) of every stream on the device -> uint8 [n, h, w, bands] (host),
    or into the device pointer out_ptr (packed frames)"""
    return _decode_batch(lib().vb200_jpeg_decode_batch, streams, (int(shrink),), out_ptr)


def _host_twin(fn, stream, *opts):
    """fn(stream, len, *opts, out, out_bpl, &w, &h, &bands) of a vb200_debug_*_decode: the geometry, then the pixels -> uint8
    [h, w, bands]"""
    stream = bytes(stream)
    w, h, bands = C.c_int(), C.c_int(), C.c_int()
    _check(fn(stream, len(stream), *opts, None, 0, C.byref(w), C.byref(h), C.byref(bands)))
    out = np.empty((h.value, w.value, bands.value), np.uint8)
    _check(fn(stream, len(stream), *opts, out.ctypes.data_as(C.c_void_p), w.value * bands.value, C.byref(w), C.byref(h), C.byref(bands)))
    return out


def jpeg_decode_host_twin(stream, shrink=1):
    """the decoder's per-block code compiled for the host (vb200_debug_jpeg_decode): what the CPU tests pin to libjpeg-turbo"""
    return _host_twin(lib().vb200_debug_jpeg_decode, stream, int(shrink))


def png_geometry(streams):
    """(width, height, bands) the PNG streams decode to (they must agree); no GPU needed"""
    return _batch_geometry(lib().vb200_png_decode_batch, streams)


def png_decode_batch(streams, out_ptr=None, out_bpl=None, out_frame_stride=None):
    """vips_pngload_buffer() of every stream on the device -> uint8 [n, h, w, bands] (host), or into the device pointer out_ptr
    (packed frames unless out_bpl / out_frame_stride say otherwise)"""
    return _decode_batch(lib().vb200_png_decode_batch, streams, (), out_ptr, out_bpl, out_frame_stride)


def png_decode_host_twin(stream):
    """the decoder's per-symbol / per-byte / per-pixel code compiled for the host (vb200_debug_png_decode): what the CPU tests
    pin to Pillow and zlib"""
    return _host_twin(lib().vb200_debug_png_decode, stream)


def webp_geometry(stream):
    """(width, height, bands) a lossy, still, opaque WebP stream decodes to; no GPU needed"""
    stream = bytes(stream)
    w, h, bands = C.c_int(), C.c_int(), C.c_int()
    _check(lib().vb200_webp_geometry(stream, len(stream), C.byref(w), C.byref(h), C.byref(bands)))
    return w.value, h.value, bands.value


def webp_decode_batch(streams, out_ptr=None, out_bpl=None, out_frame_stride=None, scale=1.0):
    """vips_webpload_buffer(scale=scale) of every stream (lossy, still, opaque WebP) on the device -> uint8 [n, h, w, 3] (host), or
    into the device pointer out_ptr (packed frames unless out_bpl / out_frame_stride say otherwise).  scale != 1: libwebp's
    scaled decode, the streams sharing one source size"""
    if scale == 1.0:
        return _decode_batch(lib().vb200_webp_decode_batch, streams, (), out_ptr, out_bpl, out_frame_stride)
    return _decode_batch(lib().vb200_webp_decode_batch_scaled, streams, (float(scale),), out_ptr, out_bpl, out_frame_stride)


def webp_decode_host_twin(stream, scale=1.0):
    """the decoder's per-symbol / per-block / per-pixel code compiled for the host (vb200_debug_webp_decode, or at scale != 1
    vb200_debug_webp_decode_scaled with its row-streaming rescaler): what the CPU tests pin to libwebp"""
    if scale == 1.0:
        return _host_twin(lib().vb200_debug_webp_decode, stream)
    return _host_twin(lib().vb200_debug_webp_decode_scaled, stream, float(scale))


def webp_rescale_plane(plane, dst_w, dst_h, closed_form=True):
    """one uint8 plane [h, w] through libwebp's rescaler to [dst_h, dst_w] on the host (vb200_debug_webp_rescale): closed_form
    by the device kernel's per-sample function, else by the host twin's row-streaming rescaler"""
    plane = np.ascontiguousarray(plane, np.uint8)
    out = np.empty((dst_h, dst_w), np.uint8)
    _check(lib().vb200_debug_webp_rescale(plane.ctypes.data_as(C.c_void_p), plane.shape[1], plane.shape[1], plane.shape[0], int(dst_w),
                                          int(dst_h), int(closed_form), out.ctypes.data_as(C.c_void_p), int(dst_w)))
    return out


def webp_times():
    """{kernel: device ms} of the last WebP batch on this thread (header, tokens, recon, rgb), measured only with VB200_WEBP_TIMING
    set in the environment; None without it"""
    ms = (C.c_float * 4)()
    lib().vb200_debug_webp_times(ms)
    return None if ms[0] < 0 else dict(zip(("header", "tokens", "recon", "rgb"), [round(v, 3) for v in ms]))


def webp_tables():
    """the VP8 constant tables as the decoder holds them, as one bytes object (see vb200_debug_webp_tables)"""
    n = C.c_size_t()
    _check(lib().vb200_debug_webp_tables(None, 0, C.byref(n)))
    buf = C.create_string_buffer(n.value)
    _check(lib().vb200_debug_webp_tables(buf, n.value, C.byref(n)))
    return buf.raw


def gif_geometry(stream):
    """(width, height, bands, frames) of a GIF stream after libnsgif's scan (the screen, not the pages); no GPU needed"""
    stream = bytes(stream)
    w, h, bands, frames = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    _check(lib().vb200_gif_geometry(stream, len(stream), C.byref(w), C.byref(h), C.byref(bands), C.byref(frames)))
    return w.value, h.value, bands.value, frames.value


def _gif_batch_geometry(b, page, n):
    return _batch_geometry(lib().vb200_gif_decode_batch, b, int(page), int(n))


def gif_decode_batch(streams, page=0, n=1, out_ptr=None, out_bpl=None, out_frame_stride=None):
    """vips_gifload_buffer(page=page, n=n) of every stream on the device -> uint8 [streams, h * pages, w, bands] (host), or
    into the device pointer out_ptr (packed unless out_bpl / out_frame_stride say otherwise)"""
    return _decode_batch(lib().vb200_gif_decode_batch, streams, (int(page), int(n)), out_ptr, out_bpl, out_frame_stride)


def gif_decode_host_twin(stream, page=0, n=1):
    """the decoder's per-code / per-pixel code compiled for the host (vb200_debug_gif_decode): what the CPU tests pin to
    libnsgif -> uint8 [h * pages, w, bands]"""
    return _host_twin(lib().vb200_debug_gif_decode, stream, int(page), int(n))


def tiff_geometry(stream, page=0, subifd=-1):
    """(width, height, bands, pages, subifds) of the TIFF IFD page / subifd select: the stream's page count and the SubIFD count
    of that page's main IFD; no GPU needed"""
    stream = bytes(stream)
    v = [C.c_int() for _ in range(5)]
    _check(lib().vb200_tiff_geometry(stream, len(stream), int(page), int(subifd), *[C.byref(x) for x in v]))
    return tuple(x.value for x in v)


def tiff_decode_batch(streams, page=0, n=1, subifd=-1, out_ptr=None, out_bpl=None, out_frame_stride=None):
    """vips_tiffload_buffer(page=page, n=n, subifd=subifd) of every stream on the device -> uint8 [streams, h * pages, w, bands]
    (host), or into the device pointer out_ptr (packed unless out_bpl / out_frame_stride say otherwise)"""
    return _decode_batch(lib().vb200_tiff_decode_batch, streams, (int(page), int(n), int(subifd)), out_ptr, out_bpl, out_frame_stride)


def tiff_decode_host_twin(stream, page=0, n=1, subifd=-1):
    """the decoder's per-code / per-byte code compiled for the host (vb200_debug_tiff_decode) -> uint8 [h * pages, w, bands]"""
    return _host_twin(lib().vb200_debug_tiff_decode, stream, int(page), int(n), int(subifd))


def tiff_icc_profile(stream, page=0, subifd=-1):
    """the ICCProfile tag of the TIFF IFD page / subifd select (bytes, or None)"""
    return _icc_blob(lib().vb200_tiff_icc_profile, stream, int(page), int(subifd))


def tiff_lzw_host_twin(data, want):
    """one TIFF LZW segment (libtiff's new-style codes) through the decoder's LZW on the host -> exactly `want` bytes; vb.Error
    when libtiff would refuse it or it holds fewer"""
    data = bytes(data)
    out = C.create_string_buffer(max(1, int(want)))
    n = C.c_size_t()
    _check(lib().vb200_debug_tiff_lzw(data, len(data), int(want), out, C.byref(n)))
    return out.raw[:n.value]


def thumbnail_tiff_level(stream, width, height=None, size="both"):
    """(subifd, page) vips_thumbnail_buffer loads from a TIFF for this thumbnail: a pyramid level, or (-1, 0); no GPU needed"""
    stream = bytes(stream)
    sub, page = C.c_int(), C.c_int()
    _check(lib().vb200_thumbnail_tiff_level(stream, len(stream), int(width), int(height or 0), SIZES[size], C.byref(sub), C.byref(page)))
    return sub.value, page.value


def thumbnail_pyramid_level(input_width, input_height, pages, subifds, width, height=None, size="both"):
    """the level choice of thumbnail_tiff_level over given geometries: pages / subifds are lists of (width, height), pages[0]
    being the main image -> (subifd, page); no GPU needed"""
    pw = (C.c_int * max(1, len(pages)))(*[p[0] for p in pages])
    ph = (C.c_int * max(1, len(pages)))(*[p[1] for p in pages])
    sw = (C.c_int * max(1, len(subifds)))(*[p[0] for p in subifds])
    sh = (C.c_int * max(1, len(subifds)))(*[p[1] for p in subifds])
    sub, page = C.c_int(), C.c_int()
    _check(lib().vb200_debug_thumbnail_pyramid_level(int(input_width), int(input_height), len(pages), pw, ph, len(subifds), sw, sh,
                                                     int(width), int(height or 0), SIZES[size], C.byref(sub), C.byref(page)))
    return sub.value, page.value


def lzw_host_twin(data, min_code_size, want, lenient=False):
    """GIF LZW data (sub-blocks joined) through the GIF decoder's LZW on the host -> at most `want` index bytes; vb.Error
    for a code libnsgif refuses (lenient: the rule of its complex path, which takes a bad code at a multiple of 4096 values
    as the end)"""
    data = bytes(data)
    out = C.create_string_buffer(max(1, int(want)))
    n = C.c_size_t()
    _check(lib().vb200_debug_lzw(data, len(data), int(min_code_size), int(want), int(bool(lenient)), out, C.byref(n)))
    return out.raw[:n.value]


def inflate_host_twin(data, cap=1 << 24):
    """raw deflate data (RFC 1951, no zlib header) through the PNG decoder's inflate on the host -> bytes; vb.Error when it
    refuses the stream or the output would exceed cap bytes"""
    data = bytes(data)
    out = C.create_string_buffer(max(1, cap))
    n = C.c_size_t()
    _check(lib().vb200_debug_inflate(data, len(data), out, cap, C.byref(n)))
    return out.raw[:n.value]


def rank_host_twin(a, width, height, index):
    """rank.cu's tile staging + radix select compiled for the host (vb200_debug_rank_host): what the CPU tests pin to rank.c"""
    a = np.ascontiguousarray(a)
    if a.ndim == 2:
        a = a[:, :, None]
    out = np.empty_like(a)
    _check(lib().vb200_debug_rank_host(a.ctypes.data_as(C.c_void_p), a.shape[1], a.shape[0], a.shape[2], FORMATS[a.dtype], int(width),
                                       int(height), int(index), out.ctypes.data_as(C.c_void_p)))
    return out


def hist_local_host_twin(a, width, height, max_slope=0, staged=None):
    """histogram.cu's hist_local staging, window update and element arithmetic compiled for the host
    (vb200_debug_hist_local_host): what the CPU tests pin to hist_local.c.  staged: None as planned, else forced on / off"""
    a = np.ascontiguousarray(a, np.uint8)
    if a.ndim == 2:
        a = a[:, :, None]
    out = np.empty_like(a)
    _check(lib().vb200_debug_hist_local_host(a.ctypes.data_as(C.c_void_p), a.shape[1], a.shape[0], a.shape[2], int(width), int(height),
                                             int(max_slope), -1 if staged is None else int(bool(staged)),
                                             out.ctypes.data_as(C.c_void_p)))
    return out


def hist_equal_lut_host_twin(hist, dtype):
    """hist_equal's LUT from a (width, n_bands) uint32 histogram, through histogram.cu's per-entry arithmetic compiled for the
    host (vb200_debug_hist_equal_lut_host) -> (width, n_bands) array of dtype (uint8 or uint16)"""
    h = np.asarray(hist, np.uint32)
    if h.ndim == 1:
        h = h[:, None]
    band_major = np.ascontiguousarray(h.T)
    lut = np.empty(band_major.shape, np.dtype(dtype))
    _check(lib().vb200_debug_hist_equal_lut_host(band_major.ctypes.data_as(C.c_void_p), h.shape[0], h.shape[1], FORMATS[np.dtype(dtype)],
                                                 lut.ctypes.data_as(C.c_void_p)))
    return np.ascontiguousarray(lut.T)


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


def _save_batch(fn, opts, frames, in_ptr, shape, stride, extra=()):
    """the body of jpegsave_batch / pngsave_batch: fn(src, where, bpl, frame_stride, n, w, h, bands, opts, *extra, out, HOST,
    stride, lens) over frames on the host or at in_ptr, the streams into one reused host array -> list of bytes.  stride:
    bytes per output slot, or a function of (w, h, bands) that gives it"""
    if in_ptr is None:
        frames = np.ascontiguousarray(frames)
        if frames.ndim == 3:
            frames = frames[..., None]
        n, h, w, bands = frames.shape
        src, where = frames.ctypes.data_as(C.c_void_p), HOST
    else:
        n, h, w, bands = shape
        src, where = C.c_void_p(in_ptr), DEVICE
    stride = int(stride(w, h, bands) if callable(stride) else stride)
    out = _SAVE_BUFFERS.get((n, stride))
    if out is None:
        _SAVE_BUFFERS.clear()          # one staging array, reused: a fresh quarter gigabyte per call is all page faults
        out = _SAVE_BUFFERS[(n, stride)] = np.empty((n, stride), np.uint8)
    lens = (C.c_size_t * n)()
    _check(fn(src, where, w * bands, w * h * bands, n, w, h, bands, C.byref(opts), *extra, out.ctypes.data_as(C.c_void_p), HOST, stride, lens))
    return [out[i, :lens[i]].tobytes() for i in range(n)]


def jpegsave_batch(frames, Q=75, subsample_mode="auto", in_ptr=None, shape=None, stride=None, optimize_coding=False, restart_interval=0,
                   interlace=False):
    """vips_jpegsave_buffer() of every frame of a uint8 array [n, h, w, bands] (bands 1 or 3) on the device -> list of bytes.
    in_ptr / shape: frames already on the device (packed), shape = (n, h, w, bands).  optimize_coding: per-frame Huffman
    tables; restart_interval: an RSTn marker every that many MCUs (0..65535, 0 for none); interlace: a progressive stream
    (libjpeg's jpeg_simple_progression script, every scan with its own optimal tables)"""
    mode = {"auto": 0, "on": 1, "off": 2}[subsample_mode]
    opts = JpegSaveOptions(int(Q), mode, int(bool(optimize_coding)), int(restart_interval), int(bool(interlace)))
    return _save_batch(lib().vb200_jpegsave_batch_opts, opts, frames, in_ptr, shape, stride or (lambda w, h, bands: w * h * bands * 2 + 4096))


ADAM7 = ((0, 0, 8, 8), (4, 0, 8, 8), (0, 4, 4, 8), (2, 0, 4, 4), (0, 2, 2, 4), (1, 0, 2, 2), (0, 1, 1, 2))   # (x0, y0, dx, dy)


def _png_scan_bytes(w, h, bands, interlace=False, bitdepth=8):
    """the scanline bytes of a frame: every non-empty pass's rows, each its filter byte and its packed samples"""
    n = 0
    for x0, y0, dx, dy in (ADAM7 if interlace else ((0, 0, 1, 1),)):
        pw, ph = max(0, -(-(w - x0) // dx)), max(0, -(-(h - y0) // dy))
        if pw and ph:
            n += ph * ((pw * bands * bitdepth + 7) // 8 + 1)
    return n


def _png_stride(w, h, bands, profile, interlace=False, bitdepth=8):
    """a slot no stream of a w x h x bands frame can overflow: fixed codes cost at most 9 bits a byte"""
    n = _png_scan_bytes(w, h, bands, interlace, bitdepth or 8)
    return n + n // 8 + 400 * (n // 16383 + 2) + 12 * (n // 8192 + 2) + 2 * len(profile or b"") + 4096


def pngsave_batch(frames, compression=6, strategy="default", xres=1.0, profile=None, in_ptr=None, shape=None, stride=None, filter="none",
                  interlace=False, bitdepth=8):
    """vips_pngsave_buffer() of every frame of a uint8 array [n, h, w, bands] (bands 1-4) on the device -> list of bytes.
    in_ptr / shape: frames already on the device (packed), shape = (n, h, w, bands).  compression 4-9; strategy "default"
    or "filtered"; xres in pixels per millimetre; profile: ICC bytes written as iCCP.  stride: bytes per output slot.
    filter: "none", "sub", "up", "avg" or "paeth" (or a VipsForeignPngFilter flag), every scanline filtered with it;
    interlace: Adam7; bitdepth 1 / 2 / 4 (one band, filter none, not interlaced) or 8."""
    prof = bytes(profile) if profile else None
    return _save_batch(lib().vb200_pngsave_batch, _png_options(compression, strategy, xres, filter, interlace, bitdepth), frames, in_ptr, shape,
                       stride or (lambda w, h, bands: _png_stride(w, h, bands, prof, interlace, bitdepth)), (prof, len(prof) if prof else 0))


def pngsave_host_twin(a, compression=6, strategy="default", xres=1.0, profile=None, filter="none", interlace=False, bitdepth=8):
    """the PNG stream of one uint8 frame [h, w, bands] through the encoder's per-position, per-symbol and per-block code
    compiled for the host (vb200_debug_png_encode); no GPU"""
    a = np.ascontiguousarray(a)
    if a.ndim == 2:
        a = a[:, :, None]
    h, w, bands = a.shape
    opts = _png_options(compression, strategy, xres, filter, interlace, bitdepth)
    prof = bytes(profile) if profile else None
    n = C.c_size_t()
    args = (a.ctypes.data_as(C.c_void_p), a.strides[0], w, h, bands, C.byref(opts), prof, len(prof) if prof else 0)
    _check(lib().vb200_debug_png_encode(*args, None, 0, C.byref(n)))
    out = C.create_string_buffer(max(1, n.value))
    _check(lib().vb200_debug_png_encode(*args, out, n.value, C.byref(n)))
    return out.raw[:n.value]


def deflate_host_twin(data, level=6, strategy="default"):
    """the zlib stream (header, deflate data, Adler-32) of data at a level (4-9) and strategy through the PNG encoder's code on
    the host (vb200_debug_deflate): what zlib.compressobj(level, DEFLATED, 15, 8, strategy) gives; no GPU"""
    data = bytes(data)
    st = PNG_STRATEGIES.get(strategy, strategy)
    n = C.c_size_t()
    _check(lib().vb200_debug_deflate(data, len(data), int(level), st, None, 0, C.byref(n)))
    out = C.create_string_buffer(max(1, n.value))
    _check(lib().vb200_debug_deflate(data, len(data), int(level), st, out, n.value, C.byref(n)))
    return out.raw[:n.value]


DZ_LAYOUTS = {"dz": 0, "zoomify": 1, "google": 2, "iiif": 3, "iiif3": 4}
DZ_DEPTHS = {None: 0, "onepixel": 1, "onetile": 2, "one": 3}
DZ_CONTAINERS = {"fs": 0, "zip": 1, "szi": 2}
REGION_SHRINKS = {"mean": 0, "median": 1, "mode": 2, "max": 3, "min": 4, "nearest": 5}


class DzTile:
    """one tile of a DzPyramid: name (path relative to the directory written in), level (0 = smallest), x, y,
    rect = (left, top, width, height) in its level, bytes = its JPEG or PNG stream"""
    __slots__ = ("name", "level", "x", "y", "rect", "bytes")

    def __init__(self, name, level, x, y, rect, data):
        self.name, self.level, self.x, self.y, self.rect, self.bytes = name, level, x, y, rect, data


class DzPyramid:
    """What vips_dzsave writes, in memory: .levels = [(width, height, tiles_across, tiles_down)] by the reference's level
    number (0 = smallest), .tiles (DzTile, level 0 first, then down, then across), .sidecar = (name, text): the .dzi or
    ImageProperties.xml.  .write(directory) makes the tree a viewer reads."""

    def __init__(self, handle, basename):
        L = lib()
        try:
            base = None if basename is None else os.fsencode(basename)
            w, h, ta, td = C.c_int(), C.c_int(), C.c_int(), C.c_int()
            self.levels = []
            for n in range(L.vb200_dz_levels(handle)):
                _check(L.vb200_dz_level_geometry(handle, n, C.byref(w), C.byref(h), C.byref(ta), C.byref(td)))
                self.levels.append((w.value, h.value, ta.value, td.value))
            self.tiles = []
            v = [C.c_int() for _ in range(7)]
            p, n, name = C.c_void_p(), C.c_size_t(), C.create_string_buffer(4096)
            for i in range(L.vb200_dz_tiles(handle)):
                _check(L.vb200_dz_tile(handle, i, *[C.byref(x) for x in v], C.byref(p), C.byref(n)))
                _check(L.vb200_dz_tile_name(handle, i, base, name, len(name)))
                self.tiles.append(DzTile(os.fsdecode(name.value), v[0].value, v[1].value, v[2].value, tuple(x.value for x in v[3:]),
                                         C.string_at(p.value, n.value)))
            text = C.create_string_buffer(4096)
            _check(L.vb200_dz_sidecar(handle, base, name, len(name), text, len(text), C.byref(n)))
            self.sidecar = (os.fsdecode(name.value), text.raw[:n.value].decode())
        finally:
            L.vb200_dz_free(handle)

    def write(self, directory):
        """<directory>/<basename>.dzi + <basename>_files/<level>/<x>_<y><suffix>, or the zoomify tree"""
        for name, data in [(t.name, t.bytes) for t in self.tiles] + [(self.sidecar[0], self.sidecar[1].encode())]:
            path = os.path.join(directory, name)
            os.makedirs(os.path.dirname(path), exist_ok=True)
            with open(path, "wb") as f:
                f.write(data)


def _dz_image(image, in_ptr, shape, bpl):
    """(CImage, keep-alive) of a host array / Image, or of device memory in_ptr with shape = (height, width, bands)"""
    if in_ptr is not None:
        h, w, bands = shape
        return CImage(w, h, bands, 0, 1 if bands < 3 else 22, DEVICE, C.c_void_p(in_ptr), int(bpl or w * bands)), None
    a = image.array if isinstance(image, Image) else np.asarray(image)
    if a.ndim == 2:
        a = a[:, :, None]
    if a.dtype not in FORMATS:
        raise Error("unsupported dtype %s" % a.dtype)
    if a.strides[1:] != (a.shape[2] * a.itemsize, a.itemsize) or a.strides[0] < a.shape[1] * a.shape[2] * a.itemsize:
        a = np.ascontiguousarray(a)
    return CImage(a.shape[1], a.shape[0], a.shape[2], FORMATS[a.dtype], 1 if a.shape[2] < 3 else 22, HOST, C.c_void_p(a.ctypes.data),
                  a.strides[0]), a


def _dzsave(fn, image, basename, layout, tile_size, overlap, depth, Q, suffix, region_shrink, skip_blanks, container, subsample_mode,
            optimize_coding, restart_interval, interlace, in_ptr, shape, bpl, png=None):
    """fn(image, DzOptions, [png,] &handle) -> DzPyramid; png: the PngSaveOptions of vb200_dzsave_png"""
    pick = lambda table, v: table[v] if v in table else int(v)
    jpeg = JpegSaveOptions(int(Q), {"auto": 0, "on": 1, "off": 2}[subsample_mode], int(bool(optimize_coding)), int(restart_interval),
                           int(bool(interlace)))
    opts = DzOptions(pick(DZ_LAYOUTS, layout), int(tile_size or 0), -1 if overlap is None else int(overlap), pick(DZ_DEPTHS, depth),
                     pick(REGION_SHRINKS, region_shrink), int(skip_blanks) + 1, pick(DZ_CONTAINERS, container),
                     None if suffix is None else suffix.encode(), jpeg)
    cin, keep = _dz_image(image, in_ptr, shape, bpl)
    handle = C.c_void_p()
    _check(fn(C.byref(cin), C.byref(opts), *(() if png is None else (C.byref(png),)), C.byref(handle)))
    return DzPyramid(handle, basename)


def dzsave(image, basename=None, layout="dz", tile_size=None, overlap=None, depth=None, Q=75, suffix=None, region_shrink="mean",
           skip_blanks=-1, container="fs", subsample_mode="auto", optimize_coding=False, restart_interval=0, interlace=False, in_ptr=None,
           shape=None, bpl=None):
    """vips_dzsave on the device: the Deep Zoom ("dz") or Zoomify pyramid of a uint8 image of 1 or 3 bands, every level and
    every JPEG tile made by CUDA kernels -> DzPyramid.  image: an H x W x bands array or Image on the host, or None with
    in_ptr / shape = (height, width, bands) / bpl for pixels already on the device.  tile_size / overlap / depth None: the
    layout's defaults.  The remaining options are the reference's; what the device path does not take raises Error."""
    return _dzsave(lib().vb200_dzsave, image, basename, layout, tile_size, overlap, depth, Q, suffix, region_shrink, skip_blanks, container,
                   subsample_mode, optimize_coding, restart_interval, interlace, in_ptr, shape, bpl)


def dzsave_host_twin(image, basename=None, layout="dz", tile_size=None, overlap=None, depth=None, Q=75, suffix=None, region_shrink="mean",
                     skip_blanks=-1, container="fs", subsample_mode="auto", optimize_coding=False, restart_interval=0, interlace=False):
    """dzsave through the kernels' per-pixel code and the encoder's host twin on the CPU (vb200_debug_dzsave): no GPU"""
    return _dzsave(lib().vb200_debug_dzsave, image, basename, layout, tile_size, overlap, depth, Q, suffix, region_shrink, skip_blanks,
                   container, subsample_mode, optimize_coding, restart_interval, interlace, None, None, None)


def dzsave_png(image, basename=None, layout="dz", tile_size=None, overlap=None, depth=None, suffix=None, compression=6, strategy="default",
               filter="none", interlace=False, bitdepth=8, xres=1.0, region_shrink="mean", skip_blanks=-1, container="fs", in_ptr=None, shape=None,
               bpl=None):
    """vips_dzsave with suffix ".png" on the device: the Deep Zoom ("dz") or Zoomify pyramid of a uint8 image of 1 to 4 bands
    with PNG tiles, every level and every tile's deflate made by CUDA kernels -> DzPyramid.  2 and 4 bands are grey / RGB with
    alpha, and their levels are alpha-weighted (vips_region_shrink_alpha).  suffix None is ".png"; compression, strategy,
    filter, interlace, bitdepth and xres are pngsave_batch's.  image / in_ptr / shape / bpl and the layout options as in
    dzsave(); what the device path does not take raises Error."""
    return _dzsave(lib().vb200_dzsave_png, image, basename, layout, tile_size, overlap, depth, 75, suffix, region_shrink, skip_blanks, container,
                   "auto", False, 0, False, in_ptr, shape, bpl, _png_options(compression, strategy, xres, filter, interlace, bitdepth))


def dzsave_png_host_twin(image, basename=None, layout="dz", tile_size=None, overlap=None, depth=None, suffix=None, compression=6,
                         strategy="default", filter="none", interlace=False, bitdepth=8, xres=1.0, region_shrink="mean", skip_blanks=-1,
                         container="fs"):
    """dzsave_png through the kernels' per-pixel code and the PNG encoder's host twin on the CPU (vb200_debug_dzsave_png): no GPU"""
    return _dzsave(lib().vb200_debug_dzsave_png, image, basename, layout, tile_size, overlap, depth, 75, suffix, region_shrink, skip_blanks,
                   container, "auto", False, 0, False, None, None, None, _png_options(compression, strategy, xres, filter, interlace, bitdepth))


def dz_pyramid_level(image, n_from_top, in_ptr=None, shape=None, bpl=None):
    """level n_from_top of the pixel pyramid dzsave cuts its tiles from (0 = the image, 1 = half size ...), on the device ->
    uint8 array [height, width, bands] on the host.  2 and 4 bands are shrunk with their alpha, as dzsave_png does"""
    cin, keep = _dz_image(image, in_ptr, shape, bpl)
    cout = CImage()
    if in_ptr is not None:
        import torch
        w, h = cin.Xsize, cin.Ysize
        for _ in range(int(n_from_top)):
            w, h = (w + 1) // 2, (h + 1) // 2
        rows = torch.empty((h, w * cin.Bands), dtype=torch.uint8, device="cuda")     # the op fills the caller's buffer
        cout.data, cout.bpl = rows.data_ptr(), w * cin.Bands
        _check(lib().vb200_dz_pyramid_level(C.byref(cin), int(n_from_top), C.byref(cout)))
        return rows.cpu().numpy().reshape(cout.Ysize, cout.Xsize, cout.Bands)
    _check(lib().vb200_dz_pyramid_level(C.byref(cin), int(n_from_top), C.byref(cout)))
    buf = (C.c_uint8 * (cout.Ysize * cout.bpl)).from_address(cout.data)
    arr = np.frombuffer(buf, np.uint8).reshape(cout.Ysize, cout.Xsize, cout.Bands).copy()
    lib().vb200_image_free(C.byref(cout))
    return arr


def dz_pyramid_level_host_twin(image, n_from_top):
    """the same level through the kernel's per-pixel code on the CPU (vb200_debug_dz_pyramid_level): no GPU"""
    cin, keep = _dz_image(image, None, None, None)
    w, h = cin.Xsize, cin.Ysize
    for _ in range(int(n_from_top)):
        w, h = (w + 1) // 2, (h + 1) // 2
    out = np.empty((h, w, cin.Bands), np.uint8)
    _check(lib().vb200_debug_dz_pyramid_level(cin.data, cin.bpl, cin.Xsize, cin.Ysize, cin.Bands, int(n_from_top), out.ctypes.data_as(C.c_void_p)))
    return out


def _thumbnail_buffer_pages(stream, width, height, size, icc, linear, page, n):
    """vb200_thumbnail_buffer_pages -> (uint8 array, page height of the result or None for one page)"""
    out = CImage()
    out.where = HOST
    oph = C.c_int()
    _check(lib().vb200_thumbnail_buffer_pages(stream, len(stream), C.byref(out), int(width), int(height or 0), SIZES[size],
                                              C.byref(icc) if icc is not None else None, int(linear), int(page), int(n), C.byref(oph)))
    a = Image._take(out).array
    return a, (oph.value if oph.value < a.shape[0] else None)


def _is_webp(stream):
    return len(stream) >= 12 and stream[:4] == b"RIFF" and stream[8:12] == b"WEBP"


def _thumbnail_webp_buffer(stream, width, height, size, icc, linear):
    """vb200_thumbnail_webp_buffer: a WebP stream loaded at vips_thumbnail's scale, then thumbnailed -> uint8 array"""
    out = CImage()
    out.where = HOST
    _check(lib().vb200_thumbnail_webp_buffer(stream, len(stream), C.byref(out), int(width), int(height or 0), SIZES[size],
                                             C.byref(icc) if icc is not None else None, int(linear)))
    return Image._take(out).array


def thumbnail_buffer(stream, width, height=None, size="both", output_profile=None, input_profile=None, intent="relative",
                     builtin_profiles=None, page=0, n=1, return_page_height=False):
    """vips_thumbnail_buffer() of a JPEG, PNG, GIF, TIFF or WebP stream: decode (JPEG with shrink-on-load, WebP at
    thumbnail_webp_scale's scale, GIF's pages page .. page + n - 1, n = -1 for all from page on, a TIFF's pyramid level as
    thumbnail_tiff_level picks it) + thumbnail on the device -> uint8 array; with output_profile, colour-managed with the profile
    the stream embeds (APP2 ICC_PROFILE or iCCP; GIF has none).  PNG streams with eXIf are refused: their orientation would
    need vips_autorot.  A GIF of several pages thumbnails as a page strip; return_page_height=True returns
    (array, page height) with None for a result of one page"""
    stream = bytes(stream)
    icc = thumbnail_icc(output_profile, input_profile, intent, builtin_profiles)
    if return_page_height or page != 0 or n != 1:
        a, ph = _thumbnail_buffer_pages(stream, width, height, size, icc, False, page, n)
        return (a, ph) if return_page_height else a
    if _is_webp(stream):
        return _thumbnail_webp_buffer(stream, width, height, size, icc, False)
    out = CImage()
    out.where = HOST
    if icc is None:
        _check(lib().vb200_thumbnail_buffer(stream, len(stream), C.byref(out), int(width), int(height or 0), SIZES[size]))
    else:
        _check(lib().vb200_thumbnail_buffer_icc(stream, len(stream), C.byref(out), int(width), int(height or 0), SIZES[size],
                                                C.byref(icc)))
    return Image._take(out).array


def thumbnail_buffer_linear(stream, width, height=None, size="both", output_profile=None, input_profile=None, intent="relative",
                            builtin_profiles=None, page=0, n=1, return_page_height=False):
    """vips_thumbnail_buffer(linear=TRUE) of a JPEG, PNG, GIF or WebP stream: full-size decode (WebP at thumbnail_webp_scale's
    scale, which applies in linear mode too) + linear-light thumbnail on the device,
    colour-managed with the profile the stream embeds and / or the profiles given.  PNG streams with eXIf are refused.
    page / n / return_page_height as thumbnail_buffer"""
    stream = bytes(stream)
    icc = linear_icc(output_profile, input_profile, intent, builtin_profiles)
    if return_page_height or page != 0 or n != 1:
        a, ph = _thumbnail_buffer_pages(stream, width, height, size, icc, True, page, n)
        return (a, ph) if return_page_height else a
    if _is_webp(stream):
        return _thumbnail_webp_buffer(stream, width, height, size, icc, True)
    out = CImage()
    out.where = HOST
    _check(lib().vb200_thumbnail_buffer_linear_icc(stream, len(stream), C.byref(out), int(width), int(height or 0), SIZES[size],
                                                   C.byref(icc)))
    return Image._take(out).array


def thumbnail_webp_scale(width, height, target_width, target_height=None, size="both"):
    """vips_thumbnail_open's WebP load (thumbnail.c:627-636): (scale, scaled width, scaled height) webpload is asked for"""
    sc, sw, sh = C.c_double(), C.c_int(), C.c_int()
    _check(lib().vb200_thumbnail_webp_scale(int(width), int(height), int(target_width), int(target_height or 0), SIZES[size], C.byref(sc),
                                            C.byref(sw), C.byref(sh)))
    return sc.value, sw.value, sh.value


def thumbnail_jpegshrink(width, height, target_width, target_height=None, size="both"):
    """vips_thumbnail_find_jpegshrink (thumbnail.c:489-517)"""
    return int(lib().vb200_thumbnail_jpegshrink(width, height, target_width, target_height or 0, SIZES[size]))


def thumbnail_pages_size(width, page_height, n_pages, target_width, target_height=None, size="both"):
    """(hshrink, vshrink, out_width, out_height, out_page_height) a plan for a strip of n_pages pages computes
    (vb200_debug_thumbnail_pages_size, no GPU needed), or None where the plan declines"""
    hs, vs, ow, oh, oph = C.c_double(), C.c_double(), C.c_int(), C.c_int(), C.c_int()
    if lib().vb200_debug_thumbnail_pages_size(int(width), int(page_height), int(n_pages), int(target_width), int(target_height or 0),
                                              SIZES[size], C.byref(hs), C.byref(vs), C.byref(ow), C.byref(oh), C.byref(oph)):
        lib().vb200_error_clear()
        return None
    return hs.value, vs.value, ow.value, oh.value, oph.value


def thumbnail_pages_kernel(width, page_height, n_pages, bands, target_width, target_height=None, size="both", has_alpha=None):
    """the kernel name (ThumbnailPlan.kernel) of the plan for a strip of n_pages pages, planned without a GPU; None where the
    plan declines"""
    if has_alpha is None:
        has_alpha = bands == 2 or bands >= 4
    name = C.create_string_buffer(256)
    if lib().vb200_debug_thumbnail_pages_kernel(int(width), int(page_height), int(n_pages), int(bands), int(has_alpha), int(target_width),
                                                int(target_height or 0), SIZES[size], name, 256):
        lib().vb200_error_clear()
        return None
    return name.value.decode()


class ThumbnailPlan:
    """The batched tile pump (vb200_thumbnail_plan_* in include/vb200.h)."""

    def __init__(self, width, height, bands=4, target_width=512, target_height=None, size="both",
                 has_alpha=None, linear=False, page_height=None):
        """height: the frame's height, a whole strip of pages of page_height rows when page_height is set (read as
        vips_image_get_page_height does: one page unless it is below height and divides it)"""
        if has_alpha is None:
            # vips_image_hasalpha for the interpretation Image() guesses: B_W below 3 bands, sRGB from 3
            has_alpha = bands == 2 or bands >= 4
        self.width, self.height, self.bands = width, height, bands
        if page_height is not None and 0 < page_height < height and height % page_height == 0:
            self._p = lib().vb200_thumbnail_plan_new_pages(width, page_height, height // page_height, bands, 0, int(has_alpha),
                                                           target_width, target_height or 0, SIZES[size], int(linear))
        else:
            self._p = lib().vb200_thumbnail_plan_new(width, height, bands, 0, int(has_alpha), target_width,
                                                     target_height or 0, SIZES[size], int(linear))
        if not self._p:
            _check(-1)
        ow, oh = C.c_int(), C.c_int()
        lib().vb200_thumbnail_plan_output(self._p, C.byref(ow), C.byref(oh))
        self.out_width, self.out_height = ow.value, oh.value
        oph = int(lib().vb200_thumbnail_plan_page_height(self._p))
        self.out_page_height = oph if oph < self.out_height else None  # None: the output is one page
        self.in_frame_bytes = width * height * bands
        self.out_bands = bands
        self.out_frame_bytes = self.out_width * self.out_height * bands
        self.bytes_per_frame = int(lib().vb200_thumbnail_plan_bytes_per_frame(self._p))
        self.fused = bool(lib().vb200_thumbnail_plan_is_fused(self._p))
        self.kernel = lib().vb200_thumbnail_plan_kernel(self._p).decode()

    def set_sharpen(self, sigma=0.5, x1=2.0, y2=10.0, y3=20.0, m1=0.0, m2=3.0):
        """vips_sharpen appended to every batch of this plan (sigma <= 0: off); BASELINE config 5"""
        _check(lib().vb200_thumbnail_plan_set_sharpen(self._p, float(sigma), float(x1), float(y2), float(y3), float(m1),
                                                      float(m2)))

    def set_icc(self, output_profile=None, input_profile=None, intent="relative", builtin_profiles=None):
        """vips_thumbnail's colour management for every batch of this plan (output_profile None: off); out_bands and
        out_frame_bytes follow the output profile"""
        icc = thumbnail_icc(output_profile, input_profile, intent, builtin_profiles)
        _check(lib().vb200_thumbnail_plan_set_icc(self._p, C.byref(icc) if icc is not None else None))
        self.out_bands = int(lib().vb200_thumbnail_plan_output_bands(self._p))
        self.out_frame_bytes = self.out_width * self.out_height * self.out_bands

    def set_linear_icc(self, output_profile=None, input_profile=None, intent="relative", builtin_profiles=None, enabled=True):
        """colour management of a linear plan (thumbnail.c:766-805, 929-987): frames with an embedded profile or input_profile
        import to XYZ and export to output_profile (or to their own profile); others export to output_profile if set, else
        run the plain path.  enabled=False: off"""
        icc = linear_icc(output_profile, input_profile, intent, builtin_profiles) if enabled else None
        _check(lib().vb200_thumbnail_plan_set_linear_icc(self._p, C.byref(icc) if icc is not None else None))
        self.out_bands = int(lib().vb200_thumbnail_plan_output_bands(self._p))
        self.out_frame_bytes = self.out_width * self.out_height * self.out_bands

    def close(self):
        if self._p:
            lib().vb200_thumbnail_plan_free(self._p)
            self._p = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def run_device(self, in_ptr, out_ptr, n_frames, in_stride=None, out_stride=None, embedded=None):
        """Device pointers (ints); queued on the stream set with set_stream().  embedded: each frame's ICC profile
        (bytes or None) for the colour-management stage"""
        if embedded is None:
            _check(lib().vb200_thumbnail_batch_device(self._p, C.c_void_p(in_ptr), in_stride or self.in_frame_bytes,
                                                      C.c_void_p(out_ptr), out_stride or self.out_frame_bytes,
                                                      n_frames))
            return
        keep, ptrs, lens = _embedded_arrays(embedded, n_frames)
        _check(lib().vb200_thumbnail_batch_device_icc(self._p, C.c_void_p(in_ptr), in_stride or self.in_frame_bytes,
                                                      C.c_void_p(out_ptr), out_stride or self.out_frame_bytes, n_frames,
                                                      ptrs, lens))

    def run_host_ptr(self, in_ptr, out_ptr, n_frames, embedded=None):
        if embedded is None:
            _check(lib().vb200_thumbnail_batch_host(self._p, C.c_void_p(in_ptr), self.in_frame_bytes,
                                                    C.c_void_p(out_ptr), self.out_frame_bytes, n_frames))
            return
        keep, ptrs, lens = _embedded_arrays(embedded, n_frames)
        _check(lib().vb200_thumbnail_batch_host_icc(self._p, C.c_void_p(in_ptr), self.in_frame_bytes, C.c_void_p(out_ptr),
                                                    self.out_frame_bytes, n_frames, ptrs, lens))

    def _run_streams(self, fn, streams, opts, out_ptr):
        b = streams if isinstance(streams, StreamBatch) else StreamBatch(streams)
        if out_ptr is not None:
            _check(fn(self._p, b.ptrs, b.lens, b.n, *opts, C.c_void_p(out_ptr), DEVICE, self.out_frame_bytes))
            return None
        out = np.empty((b.n, self.out_height, self.out_width, self.out_bands), np.uint8)
        _check(fn(self._p, b.ptrs, b.lens, b.n, *opts, out.ctypes.data_as(C.c_void_p), HOST, self.out_frame_bytes))
        return out

    def run_jpeg(self, streams, shrink, out_ptr=None):
        """JPEG streams decoded at `shrink` on the device and thumbnailed by this plan (made for the decoded
        geometry): -> uint8 [n, OH, OW, bands] on the host, or into the device pointer out_ptr"""
        return self._run_streams(lib().vb200_thumbnail_plan_run_jpeg, streams, (int(shrink),), out_ptr)

    def run_webp(self, streams, scale, out_ptr=None):
        """WebP streams decoded on the device at webpload's `scale` and thumbnailed by this plan (made for the scaled
        geometry): -> uint8 [n, OH, OW, bands] on the host, or into the device pointer out_ptr"""
        return self._run_streams(lib().vb200_thumbnail_plan_run_webp, streams, (float(scale),), out_ptr)

    def run_png(self, streams, out_ptr=None):
        """PNG streams decoded on the device at full size and thumbnailed by this plan (made for the decoded geometry):
        -> uint8 [n, OH, OW, bands] on the host, or into the device pointer out_ptr"""
        return self._run_streams(lib().vb200_thumbnail_plan_run_png, streams, (), out_ptr)

    def run_tiff(self, streams, out_ptr=None, page=0, n=1, subifd=-1):
        """vb200_thumbnail_plan_run_tiff: the streams' pages page .. page + n - 1 at subifd through the plan"""
        return self._run_streams(lib().vb200_thumbnail_plan_run_tiff, streams, (int(page), int(n), int(subifd)), out_ptr)

    def run_gif(self, streams, out_ptr=None, page=0, n=1):
        """GIF streams, pages page .. page + n - 1 of each (n = -1: every page from page on) decoded on the device at full size
        and thumbnailed by this plan (made for the screen, or with page_height = the screen height for a strip of several
        pages; 3 or 4 bands): -> uint8 [n, OH, OW, bands] on the host, or into the device pointer out_ptr"""
        return self._run_streams(lib().vb200_thumbnail_plan_run_gif_pages, streams, (int(page), int(n)), out_ptr)

    def run_host(self, frames, embedded=None):
        """frames: uint8 array [n, H, W, bands] in host memory -> [n, OH, OW, out_bands]."""
        frames = np.ascontiguousarray(frames)
        assert frames.dtype == np.uint8 and frames.shape[1:] == (self.height, self.width, self.bands)
        out = np.empty((frames.shape[0], self.out_height, self.out_width, self.out_bands), np.uint8)
        self.run_host_ptr(frames.ctypes.data, out.ctypes.data, frames.shape[0], embedded)
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

    def hist_find(self, band=-1):
        _check(lib().vb200_chain_add_hist_find(self._p, int(band)))
        return self

    def hist_equal(self, band=-1):
        _check(lib().vb200_chain_add_hist_equal(self._p, int(band)))
        return self

    def hist_local(self, width, height, max_slope=0):
        _check(lib().vb200_chain_add_hist_local(self._p, int(width), int(height), int(max_slope)))
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

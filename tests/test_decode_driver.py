"""The decoders' shared driver (csrc/decode.cu): vb200_{jpeg,png,gif,tiff,webp}_decode_batch and the matching *load_buffer
entry points behave alike -- errors that name the stream, one geometry per batch, host and device delivery, batch-or-nothing into host
memory, and one interpretation rule for the loaders."""
import ctypes as C
import io
import re

import numpy as np
import pytest
from PIL import Image as PIL

import libvips_b200 as vb

RNG = np.random.default_rng(41)


def _jpeg(h, w, bands):
    a = RNG.integers(0, 256, (h, w, bands), dtype=np.uint8)
    b = io.BytesIO()
    PIL.fromarray(a[:, :, 0] if bands == 1 else a).save(b, "JPEG", quality=90)
    return b.getvalue()


def _png(h, w, bands):
    a = RNG.integers(0, 256, (h, w, bands), dtype=np.uint8)
    b = io.BytesIO()
    PIL.fromarray(a[:, :, 0] if bands == 1 else a).save(b, "PNG")
    return b.getvalue()


def _gif(h, w, bands):
    a = RNG.integers(0, 256, (h, w, 3), dtype=np.uint8)
    b = io.BytesIO()
    # a transparent index gives nsgifload's 4 bands
    PIL.fromarray(a).quantize(32).save(b, "GIF", **({"transparency": 3} if bands == 4 else {}))
    return b.getvalue()


def _tiff(h, w, bands):
    a = RNG.integers(0, 256, (h, w, bands), dtype=np.uint8)
    b = io.BytesIO()
    PIL.fromarray(a[:, :, 0] if bands == 1 else a).save(b, "TIFF", compression="tiff_lzw")
    return b.getvalue()


def _webp(h, w, bands):
    a = RNG.integers(0, 256, (h, w, bands), dtype=np.uint8)
    b = io.BytesIO()
    PIL.fromarray(a).save(b, "WEBP", quality=80)
    return b.getvalue()


MAKE = {"jpeg": _jpeg, "png": _png, "gif": _gif, "tiff": _tiff, "webp": _webp}
BANDS = {"jpeg": (1, 3), "png": (1, 2, 3, 4), "gif": (3, 4), "tiff": (1, 2, 3, 4), "webp": (3,)}
NOUN = {"jpeg": "frame", "png": "frame", "gif": "stream", "tiff": "frame", "webp": "frame"}
DOMAIN = {"jpeg": "jpeg_decode_batch", "png": "png_decode_batch", "gif": "gif_decode_batch", "tiff": "tiff_decode_batch",
          "webp": "webp_decode_batch"}


def _opts(fmt):
    return {"jpeg": (1,), "png": (), "gif": (0, 1), "tiff": (0, 1, -1), "webp": ()}[fmt]


def _fn(fmt):
    return getattr(vb.lib(), "vb200_%s_decode_batch" % fmt)


def _call(fmt, streams, out, location, bpl, stride):
    """rc, error text of vb200_<fmt>_decode_batch"""
    b = vb.StreamBatch(streams)
    w, h, bands = C.c_int(), C.c_int(), C.c_int()
    rc = _fn(fmt)(b.ptrs, b.lens, b.n, *_opts(fmt), out, location, bpl, stride, C.byref(w), C.byref(h), C.byref(bands))
    err = vb.lib().vb200_error_buffer().decode()
    vb.lib().vb200_error_clear()
    return rc, err, (w.value, h.value, bands.value)


def _corrupt_header(fmt, s):
    return s[:12] if fmt == "gif" else s[:24]


# -------------------------------------------------------------------------------------------------------- without a device

@pytest.mark.parametrize("fmt", sorted(MAKE))
def test_geometry_names_the_stream(fmt):
    good = MAKE[fmt](20, 30, 3)
    rc, err, _ = _call(fmt, [good, _corrupt_header(fmt, good), good], None, vb.HOST, 0, 0)
    assert rc == -1 and re.search(r"%s 1: \S" % NOUN[fmt], err), err
    assert err.count(DOMAIN[fmt]) == 1, err


@pytest.mark.parametrize("fmt", sorted(MAKE))
def test_geometry_of_a_batch(fmt):
    a, b = MAKE[fmt](20, 30, 3), MAKE[fmt](21, 30, 3)
    assert _call(fmt, [a, a], None, vb.HOST, 0, 0)[::2] == (0, (30, 20, 3))
    rc, err, _ = _call(fmt, [a, a, b], None, vb.HOST, 0, 0)
    assert rc == -1 and "one geometry" in err and "%s 2:" % NOUN[fmt] in err, err


# ---------------------------------------------------------------------------------------------------------- on the device

@pytest.mark.gpu
def test_gpu_jpeg_device_path_error_is_stated_once(vb):
    import torch
    good = _jpeg(16, 16, 3)
    bad = _corrupt_header("jpeg", good)
    with pytest.raises(vb.Error) as e:
        vb.jpeg_decode_host_twin(bad)
    reason = str(e.value).split(": ", 1)[1].strip()
    dev = torch.zeros(3 * 16 * 16 * 3, dtype=torch.uint8, device="cuda")
    rc, err, _ = _call("jpeg", [good, bad, good], C.c_void_p(dev.data_ptr()), vb.DEVICE, 48, 16 * 48)
    assert rc == -1 and err.strip() == "jpeg_decode_batch: frame 1: " + reason, err


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", sorted(MAKE))
def test_gpu_load_buffer(vb, fmt):
    for bands in BANDS[fmt]:
        s = MAKE[fmt](23, 37, bands)
        out = vb.CImage()
        out.where = vb.HOST
        name = "vb200_%sload_buffer" % fmt
        args = _opts(fmt)
        fn = getattr(vb.lib(), name)
        fn.argtypes = [C.c_void_p, C.c_size_t] + [C.c_int] * len(args) + [C.POINTER(vb.CImage)]
        vb._check(fn(s, len(s), *args, C.byref(out)))
        assert out.Type == vb.INTERPRETATIONS["b-w" if out.Bands <= 2 else "srgb"], (fmt, bands, out.Type)
        got = vb.Image._take(out).array
        want = getattr(vb, "%s_decode_batch" % fmt)([s])[0]
        assert got.shape[2] == want.shape[2] and np.array_equal(got, want), (fmt, bands)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", sorted(MAKE))
def test_gpu_host_delivery_with_strides(vb, fmt):
    import torch
    streams = [MAKE[fmt](19, 27, 3) for _ in range(3)]
    w, h, bands = vb._batch_geometry(_fn(fmt), streams, *_opts(fmt))
    line = w * bands
    dev = torch.zeros(3 * h * line, dtype=torch.uint8, device="cuda")
    assert _call(fmt, streams, C.c_void_p(dev.data_ptr()), vb.DEVICE, line, h * line)[0] == 0
    want = dev.cpu().numpy().reshape(3, h, w, bands)
    bpl, stride = line + 5, (line + 5) * h + 7
    out = np.full(3 * stride, 0xA5, np.uint8)
    assert _call(fmt, streams, out.ctypes.data_as(C.c_void_p), vb.HOST, bpl, stride)[0] == 0
    for i in range(3):
        frame = out[i * stride:i * stride + bpl * h].reshape(h, bpl)
        assert np.array_equal(frame[:, :line].reshape(h, w, bands), want[i]) and (frame[:, line:] == 0xA5).all(), (fmt, i)
    # too small a line
    rc, err, _ = _call(fmt, streams, out.ctypes.data_as(C.c_void_p), vb.HOST, line - 1, stride)
    assert rc == -1 and "output strides too small" in err, err


def _fails_in_decode(fmt):
    """a stream whose header parses and whose data the decoder refuses, and a good stream of its geometry"""
    if fmt == "gif":
        from test_gif import BAD, blocks, rand_pal, write_gif
        rng = np.random.default_rng(3)
        return BAD["past_table_50"], write_gif(50, 40, [dict(img=blocks(rng, 40, 50, 256))], rand_pal(rng, 256))
    if fmt == "tiff":
        from test_tiff import Page, img, lzw_encode, make_tiff
        a = img(24, 32, 3, 3)
        # an LZW segment that ends short of the strip's rows
        return make_tiff([Page(a, comp=5, segments=[lzw_encode(a.tobytes()[:50])])]), make_tiff([Page(a, comp=5)])
    if fmt == "webp":
        from test_webp import _cut, pillow_or_none, vp8_payload, vp8_stream
        good = vp8_stream(9000, h=30, w=30, parts=2)
        # a token partition cut short where libwebp refuses it
        return next(_cut(good, k) for k in range(len(vp8_payload(good)) - 1, 10, -1) if pillow_or_none(_cut(good, k)) is None), good
    good = MAKE[fmt](24, 32, 3)
    if fmt == "png":
        at = good.index(b"IDAT") + 4
        n = int.from_bytes(good[at - 8:at - 4], "big")
        # a deflate block of the reserved type 3
        return good[:at + 2] + b"\xff" * (n - 2) + good[at + n:], good
    sos = good.index(b"\xff\xda")
    data = sos + 2 + int.from_bytes(good[sos + 2:sos + 4], "big")
    # all-ones bits: a code no Huffman table assigns
    return good[:data] + b"\xff\x00" * ((len(good) - 2 - data) // 2) + b"\xff\xd9", good


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", sorted(MAKE))
def test_gpu_failed_host_delivery_writes_nothing(vb, fmt):
    bad, good = _fails_in_decode(fmt)
    streams = [good, bad, good]
    w, h, bands = vb._batch_geometry(_fn(fmt), streams, *_opts(fmt))
    out = np.full((3, h, w, bands), 0x5A, np.uint8)
    rc, err, _ = _call(fmt, streams, out.ctypes.data_as(C.c_void_p), vb.HOST, w * bands, w * h * bands)
    assert rc == -1 and "%s 1" % NOUN[fmt] in err, err
    assert (out == 0x5A).all()

"""WebP shrink-on-load on the device (csrc/webp.cu): vips_webpload_buffer's `scale` through libwebp's scaled decode, and WebP
thumbnails at the scale vips_thumbnail loads them.

The oracle is the libwebp inside Pillow itself, called through ctypes with options.use_scaling, the way webp2vips.c asks for
a scaled frame.  On the CPU the host twin (whose rescaler streams rows in libwebp's order) is held to it on every stream
family test_webp.py builds over a grid of output sizes; the device kernel's closed-form sample function is held to the
twin's rescaler plane by plane; and thumbnail_webp_scale to a transcription of vips_thumbnail_open's WebP factor.  On the
device every result is checked bit for bit against the twin or the oracle.
"""
import ctypes as C
import glob
import os

import numpy as np
import pytest

import libvips_b200 as vb
from test_webp import GOLDEN, PILLOW, WRITER, _cut, content, pil_webp, vp8_payload, vp8_stream  # noqa: E402

PIL = pytest.importorskip("PIL.Image")

# ------------------------------------------------------------------ libwebp through ctypes


class _Features(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("has_alpha", C.c_int), ("has_animation", C.c_int), ("format", C.c_int),
                ("pad", C.c_uint32 * 5)]


class _RGBA(C.Structure):
    _fields_ = [("rgba", C.c_void_p), ("stride", C.c_int), ("size", C.c_size_t)]


class _YUVA(C.Structure):
    _fields_ = [("y", C.c_void_p), ("u", C.c_void_p), ("v", C.c_void_p), ("a", C.c_void_p), ("y_stride", C.c_int), ("u_stride", C.c_int),
                ("v_stride", C.c_int), ("a_stride", C.c_int), ("y_size", C.c_size_t), ("u_size", C.c_size_t), ("v_size", C.c_size_t),
                ("a_size", C.c_size_t)]


class _Buf(C.Union):
    _fields_ = [("RGBA", _RGBA), ("YUVA", _YUVA)]


class _DecBuffer(C.Structure):
    _fields_ = [("colorspace", C.c_int), ("width", C.c_int), ("height", C.c_int), ("is_external_memory", C.c_int), ("u", _Buf),
                ("pad", C.c_uint32 * 4), ("private_memory", C.c_void_p)]


class _Options(C.Structure):
    _fields_ = [("bypass_filtering", C.c_int), ("no_fancy_upsampling", C.c_int), ("use_cropping", C.c_int), ("crop_left", C.c_int),
                ("crop_top", C.c_int), ("crop_width", C.c_int), ("crop_height", C.c_int), ("use_scaling", C.c_int),
                ("scaled_width", C.c_int), ("scaled_height", C.c_int), ("use_threads", C.c_int), ("dithering_strength", C.c_int),
                ("flip", C.c_int), ("alpha_dithering_strength", C.c_int), ("pad", C.c_uint32 * 5)]


class _Config(C.Structure):
    _fields_ = [("input", _Features), ("output", _DecBuffer), ("options", _Options)]


def _libwebp():
    import PIL as P
    libs = os.path.join(os.path.dirname(P.__file__), "..", "pillow.libs")
    sharp = glob.glob(os.path.join(libs, "libsharpyuv-*.so*"))
    webp = glob.glob(os.path.join(libs, "libwebp-*.so*"))
    if not sharp or not webp:
        return None
    C.CDLL(sharp[0], mode=C.RTLD_GLOBAL)
    L = C.CDLL(webp[0])
    L.WebPInitDecoderConfigInternal.argtypes = [C.POINTER(_Config), C.c_int]
    L.WebPDecode.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(_Config)]
    return L


_LIBWEBP = _libwebp()


def libwebp_scaled(stream, sw, sh):
    """WebPDecode into an external MODE_RGB buffer with use_scaling at sw x sh (None: libwebp refuses the stream)"""
    if _LIBWEBP is None:
        pytest.skip("no bundled libwebp to call")
    cfg = _Config()
    assert _LIBWEBP.WebPInitDecoderConfigInternal(C.byref(cfg), 0x0209)
    out = np.zeros((sh, sw, 3), np.uint8)
    cfg.options.use_scaling, cfg.options.scaled_width, cfg.options.scaled_height = 1, sw, sh
    cfg.output.colorspace, cfg.output.is_external_memory = 0, 1
    cfg.output.u.RGBA.rgba, cfg.output.u.RGBA.stride, cfg.output.u.RGBA.size = out.ctypes.data, sw * 3, out.size
    return out if _LIBWEBP.WebPDecode(stream, len(stream), C.byref(cfg)) == 0 else None


def webpload_size(w, h, scale):
    """webp2vips.c:513-514: rint() rounds half to even, as Python's round() does"""
    return int(round(w * scale)), int(round(h * scale))


def scale_grid(w, h):
    """scales whose output sizes straddle the filter bypass (W * 3 / 4 on one axis and on both), sit around the chroma
    width (W + 1) / 2, keep the size at scale != 1, and expand by 1.5 and 3"""
    out = set()
    for tw in {w * 3 // 4 - 1, w * 3 // 4, w * 3 // 4 + 1, (w + 1) // 2 - 1, (w + 1) // 2, (w + 1) // 2 + 1}:
        if tw >= 1:
            out.add(tw / w)
    for th in (h * 3 // 4 - 1, h * 3 // 4, h * 3 // 4 + 1):
        if th >= 1:
            out.add(th / h)
    out |= {1.0 + 0.4 / max(w, h), 1.5, 3.0, 0.37}
    return sorted(s for s in out if s != 1.0 and all(1 <= v <= 0x3FFF for v in webpload_size(w, h, s)))


# ------------------------------------------------------------------ CPU: the twin against libwebp


def _check_twin(stream, scales):
    w, h, _ = vb.webp_geometry(stream)
    for s in scales:
        sw, sh = webpload_size(w, h, s)
        want = libwebp_scaled(stream, sw, sh)
        assert want is not None, (w, h, s)
        got = vb.webp_decode_host_twin(stream, scale=s)
        assert got.shape == want.shape and np.array_equal(got, want), (w, h, s, sw, sh, int(np.abs(got.astype(int) - want).max()))


@pytest.mark.parametrize("name,stream", PILLOW, ids=[n for n, _ in PILLOW])
def test_twin_pillow_streams(name, stream):
    w, h, _ = vb.webp_geometry(stream)
    _check_twin(stream, scale_grid(w, h))


@pytest.mark.parametrize("name,stream", WRITER, ids=[n for n, _ in WRITER])
def test_twin_writer_streams(name, stream):
    w, h, _ = vb.webp_geometry(stream)
    _check_twin(stream, scale_grid(w, h))


def test_twin_fixture_and_icc():
    s = open(os.path.join(GOLDEN, "1.webp"), "rb").read()
    _check_twin(s, [0.1, 0.25, 0.5, 0.74, 0.75, 0.76, 1.001, 1.5])
    prof = open(os.path.join(os.path.dirname(GOLDEN), "profiles", "sRGB.icm"), "rb").read()
    icc = pil_webp(content("photo", 45, 61, 3), quality=80, icc_profile=prof)
    _check_twin(icc, scale_grid(61, 45))


@pytest.mark.parametrize("h,w", [(1, 1), (1, 2), (2, 1), (2, 2), (1, 37), (37, 1), (2, 41), (41, 2), (433 // 4, 301 // 4), (31, 33), (301, 433)])
def test_twin_small_and_odd_sizes(h, w):
    """W or H of 1 and 2 (where U and V are one sample wide and libwebp's special cases live), odd sizes, and the size kept
    at scale != 1 (the scaled path still runs: no upsampler, the filter as the size asks)"""
    stream = pil_webp(content("photo", h, w, h * 31 + w), quality=70)
    scales = {1.0 + 0.3 / max(w, h), 1.5, 3.0}
    for tw in range(1, min(w, 4) + 1):
        scales.add(tw / w)
    for th in range(1, min(h, 4) + 1):
        scales.add(th / h)
    _check_twin(stream, sorted(s for s in scales if s != 1.0 and min(webpload_size(w, h, s)) >= 1))


def test_same_size_differs_from_the_plain_decode():
    stream = pil_webp(content("photo", 301, 433, 5), quality=75)
    plain = vb.webp_decode_host_twin(stream)
    same = vb.webp_decode_host_twin(stream, scale=1.0 + 1e-4)
    assert same.shape == plain.shape and not np.array_equal(same, plain)
    assert np.array_equal(same, libwebp_scaled(stream, 433, 301))


def test_refusals():
    s = pil_webp(content("photo", 20, 30, 1), quality=70)
    for scale, match in ((0.01, "bad image dimensions"), (0.0, "bad image dimensions"), (-0.5, "range"), (2000.0, "range"),
                         (float("nan"), "range"), (1024.0, "bad image dimensions")):
        with pytest.raises(vb.Error, match=match):
            vb.webp_decode_host_twin(s, scale=scale)
        with pytest.raises(vb.Error, match=match):
            vb.webp_decode_batch([s], scale=scale)
    # one geometry per batch, judged on the source: two sizes that scale to one output size are still refused
    with pytest.raises(vb.Error, match="one geometry"):
        vb.webp_decode_batch([pil_webp(content("photo", 20, 30, 1)), pil_webp(content("photo", 21, 31, 1))], scale=0.5)
    # the format refusals stand at any scale
    with pytest.raises(vb.Error, match="lossless"):
        vb.webp_decode_host_twin(pil_webp(content("photo", 20, 30, 1), lossless=True), scale=0.5)


# ------------------------------------------------------------------ CPU: the closed form against the streaming rescaler


def _plane_pairs():
    """(src_w, src_h, dst_w, dst_h) of every plane the stream grids above rescale, Y and U / V"""
    pairs = set()
    for _, s in PILLOW + WRITER:
        w, h, _ = vb.webp_geometry(s)
        for sc in scale_grid(w, h):
            sw, sh = webpload_size(w, h, sc)
            pairs.add((w, h, sw, sh))
            pairs.add(((w + 1) // 2, (h + 1) // 2, sw, sh))
    for w, h in ((1, 1), (1, 2), (2, 1), (2, 2), (3, 1), (1, 3)):
        for sw in (1, 2, 3, 5):
            for sh in (1, 2, 3, 5):
                pairs.add((w, h, sw, sh))
    return sorted(pairs)


def _same_plane(sw_, sh_, dw, dh, rng):
    plane = rng.integers(0, 256, (sh_, sw_), dtype=np.uint8)
    if rng.integers(0, 4) == 0:
        plane[:] = 255
    a = vb.webp_rescale_plane(plane, dw, dh, closed_form=True)
    b = vb.webp_rescale_plane(plane, dw, dh, closed_form=False)
    assert np.array_equal(a, b), (sw_, sh_, dw, dh)


def test_closed_form_on_the_grid():
    rng = np.random.default_rng(1)
    for p in _plane_pairs():
        _same_plane(*p, rng)


def test_closed_form_random_pairs():
    """a few thousand (src, dst) pairs up to 16383 on one axis, against a small other axis"""
    rng = np.random.default_rng(2)
    for k in range(2500):
        big_s, big_d = int(rng.integers(1, 16384)), int(rng.integers(1, 16384))
        if k % 3 == 0:
            big_d = max(1, int(big_s * rng.uniform(0.01, 1.0)))
        small_s, small_d = int(rng.integers(1, 6)), int(rng.integers(1, 6))
        if big_s * max(small_s, small_d) + big_d * small_d > 3_000_000:
            big_s, big_d = max(1, big_s // 8), max(1, big_d // 8)
        if k % 2:
            _same_plane(big_s, small_s, big_d, small_d, rng)
        else:
            _same_plane(small_s, big_s, small_d, big_d, rng)


# ------------------------------------------------------------------ CPU: vips_thumbnail_open's WebP factor

SIZE_MODES = ("both", "up", "down", "force")


def py_calculate_shrink(w, h, tw, th, size):
    """thumbnail.c:405-466 without rotation or crop"""
    hs, vs = w / tw, h / th
    direction = "v" if hs < vs else "h"
    if size != "force":
        if direction == "h":
            vs = hs
        else:
            hs = vs
    if size == "up":
        hs, vs = min(1, hs), min(1, vs)
    elif size == "down":
        hs, vs = max(1, hs), max(1, vs)
    return min(hs, w), min(vs, h)


def py_webp_scale(w, h, tw, th, size):
    """thumbnail.c:468-484, 627-636 and webp2vips.c:513-514"""
    factor = max(1.0, min(py_calculate_shrink(w, h, tw, th, size)))
    scale = 1.0 / factor
    return scale, int(round(w * scale)), int(round(h * scale))


def test_thumbnail_webp_scale():
    rng = np.random.default_rng(3)
    cases = [(2048, 1536, 256, None), (550, 368, 128, 128), (100, 100, 100, None), (100, 100, 99, None), (1, 1, 1, 1), (16383, 1, 7, 3)]
    cases += [(int(rng.integers(1, 5000)), int(rng.integers(1, 5000)), int(rng.integers(1, 3000)), int(rng.integers(0, 3000)) or None)
              for _ in range(3000)]
    for w, h, tw, th in cases:
        for size in SIZE_MODES:
            got = vb.thumbnail_webp_scale(w, h, tw, th, size)
            want = py_webp_scale(w, h, tw, th or tw, size)
            assert got == want, (w, h, tw, th, size, got, want)


def test_thumbnail_buffer_keeps_its_refusal():
    s = PILLOW[3][1]
    out = vb.CImage()
    out.where = vb.HOST
    rc = vb.lib().vb200_thumbnail_buffer(s, len(s), C.byref(out), 32, 32, 0)
    msg = vb.lib().vb200_error_buffer().decode()
    vb.lib().vb200_error_clear()
    assert rc == -1 and "WebP shrink-on-load" in msg and "vb200_thumbnail_webp_buffer" in msg, msg


def test_abi():
    L = C.CDLL(vb.library_path())
    for name in ("vb200_webp_decode_batch_scaled", "vb200_webpload_buffer_scaled", "vb200_thumbnail_webp_scale", "vb200_thumbnail_webp_buffer",
                 "vb200_thumbnail_plan_run_webp", "vb200_debug_webp_decode_scaled", "vb200_debug_webp_rescale"):
        assert hasattr(L, name), name
    from libvips_b200 import _batch_geometry
    s = pil_webp(content("photo", 45, 61, 3), quality=80)
    assert _batch_geometry(vb.lib().vb200_webp_decode_batch_scaled, [s, s], 0.5) == (30, 22, 3)  # rint(22.5) is 22
    assert _batch_geometry(vb.lib().vb200_webp_decode_batch_scaled, [s], 1.0) == (61, 45, 3)


# ------------------------------------------------------------------ on the device

GPU_SCALES = (0.13, 0.5, 0.74, 0.76, 1.0001, 1.5, 3.0)


def _gpu_streams():
    return [s for _, s in PILLOW] + [s for _, s in WRITER]


@pytest.mark.gpu
def test_gpu_every_stream(vb):
    by_geometry = {}
    for s in _gpu_streams():
        by_geometry.setdefault(vb.webp_geometry(s), []).append(s)
    for (w, h, _), streams in by_geometry.items():
        for sc in GPU_SCALES + tuple(scale_grid(w, h)):
            if min(webpload_size(w, h, sc)) < 1:
                continue
            got = vb.webp_decode_batch(streams, scale=sc)
            for i, s in enumerate(streams):
                assert np.array_equal(got[i], vb.webp_decode_host_twin(s, scale=sc)), (w, h, sc, i)


def _decode_raw(streams, scale, out, location, bpl, stride):
    b = vb.StreamBatch(streams)
    ww, hh, bb = C.c_int(), C.c_int(), C.c_int()
    rc = vb.lib().vb200_webp_decode_batch_scaled(b.ptrs, b.lens, b.n, scale, C.c_void_p(out), location, bpl, stride, C.byref(ww), C.byref(hh),
                                                 C.byref(bb))
    msg = vb.lib().vb200_error_buffer().decode()
    vb.lib().vb200_error_clear()
    return rc, msg


@pytest.mark.gpu
def test_gpu_chunks(vb):
    """a batch split into chunks of 2-3 frames by the budget decodes as one, into host and device memory at padded strides, and
    a frame that fails in a later chunk is named by its index in the whole batch"""
    import torch
    h, w, scale = 37, 45, 0.6
    streams = [vp8_stream(6100 + i, h=h, w=w, parts=1 + i % 4 // 2 * 3) for i in range(9)]
    streams += [pil_webp(content("photo", h, w, 20 + i), quality=40 + 10 * i) for i in range(5)]
    want = np.stack([vb.webp_decode_host_twin(s, scale=scale) for s in streams])
    sw, sh = webpload_size(w, h, scale)
    n, bpl = len(streams), sw * 3 + 5
    stride = bpl * sh + 11
    L = vb.lib()
    try:
        L.vb200_debug_png_set_budget(40000)
        before = vb.launch_count()
        assert np.array_equal(vb.webp_decode_batch(streams, scale=scale), want)
        assert vb.launch_count() - before >= 4 * 5, "the batch did not split into chunks"
        host = np.full(stride * n, 77, np.uint8)
        rc, msg = _decode_raw(streams, scale, host.ctypes.data, vb.HOST, bpl, stride)
        assert rc == 0, msg
        dev = torch.full((stride * n,), 77, dtype=torch.uint8, device="cuda")
        rc, msg = _decode_raw(streams, scale, dev.data_ptr(), vb.DEVICE, bpl, stride)
        assert rc == 0, msg
        torch.cuda.synchronize()
        for d in (host, dev.cpu().numpy()):
            for i in range(n):
                frame = d[i * stride:i * stride + bpl * sh].reshape(sh, bpl)
                assert np.array_equal(frame[:, :sw * 3].reshape(sh, sw, 3), want[i]), i
                assert (frame[:, sw * 3:] == 77).all() and (d[i * stride + bpl * sh:(i + 1) * stride] == 77).all(), i
        cut = next(c for c in (_cut(streams[2], k) for k in range(len(vp8_payload(streams[2])) - 1, 10, -1))
                   if libwebp_scaled(c, sw, sh) is None)
        batch = streams[:11] + [cut] + streams[12:]
        host = np.full(stride * n, 0xA5, np.uint8)
        rc, msg = _decode_raw(batch, scale, host.ctypes.data, vb.HOST, bpl, stride)
        assert rc == -1 and "frame 11:" in msg, msg
        assert (host == 0xA5).all()
        rc, msg = _decode_raw(batch, scale, dev.data_ptr(), vb.DEVICE, bpl, stride)
        assert rc == -1 and "frame 11:" in msg, msg
    finally:
        L.vb200_debug_png_set_budget(0)


@pytest.mark.gpu
def test_gpu_wide_frame(vb):
    s = vp8_stream(7017, h=17, w=16383, parts=8)
    for sc in (0.3, 0.99995):  # rint(16383 * 0.99995) is 16382 while the 17 rows keep their size: Y shrinks by one column
        assert np.array_equal(vb.webp_decode_batch([s], scale=sc)[0], vb.webp_decode_host_twin(s, scale=sc)), sc


@pytest.mark.gpu
def test_gpu_webpload_and_timing(vb):
    s = pil_webp(content("photo", 120, 93, 4), quality=80)
    for sc in (0.25, 1.7):
        img = vb.Image.webpload_buffer(s, scale=sc)
        assert np.array_equal(img.numpy(), vb.webp_decode_host_twin(s, scale=sc)), sc
    assert np.array_equal(vb.Image.webpload_buffer(s).numpy(), vb.webp_decode_host_twin(s))
    os.environ["VB200_WEBP_TIMING"] = "1"
    try:
        vb.webp_decode_batch([s, s], scale=0.3)
        t = vb.webp_times()
        assert set(t) == {"header", "tokens", "recon", "rgb"} and all(v > 0 for v in t.values()), t
    finally:
        del os.environ["VB200_WEBP_TIMING"]


def _thumb_cases():
    return [(pil_webp(content("photo", 368, 550, 9), quality=80), 550, 368),
            (vp8_stream(9100, h=130, w=170, parts=2), 170, 130),
            (open(os.path.join(GOLDEN, "1.webp"), "rb").read(), 550, 368)]


@pytest.mark.gpu
def test_gpu_thumbnail_buffer(vb):
    from oracle import pyoracle
    for s, w, h in _thumb_cases():
        targets = [(128, None), (w, None), (w - 1, None), (64, 200), (200, 64), (w * 2, None)]
        for tw, th in targets:
            for size in SIZE_MODES:
                scale, _, _ = vb.thumbnail_webp_scale(w, h, tw, th, size)
                dec = vb.webp_decode_host_twin(s, scale=scale)
                try:
                    want = pyoracle.thumbnail_image(dec, tw, th, size=size)
                except ValueError:
                    # a resize up on one axis and down on the other: the thumbnail tail refuses it, as before
                    with pytest.raises(vb.Error):
                        vb.thumbnail_buffer(s, tw, th, size=size)
                    continue
                got = vb.thumbnail_buffer(s, tw, th, size=size)
                assert np.array_equal(got, want), (w, h, tw, th, size, scale)


@pytest.mark.gpu
def test_gpu_thumbnail_icc_and_linear(vb):
    """colour-managed and linear WebP thumbnails: vb200_thumbnail_image_icc / _linear_icc of the twin's scaled decode, with the
    stream's ICCP as the embedded profile"""
    profiles = os.path.join(os.path.dirname(GOLDEN), "profiles")
    srgb, p3 = (open(os.path.join(profiles, n), "rb").read() for n in ("sRGB.icm", "p3.icm"))
    builtin = {"srgb": srgb}
    for prof in (p3, srgb):
        s = pil_webp(content("photo", 150, 211, 8), quality=80, icc_profile=prof)
        assert vb.webp_icc_profile(s) == prof
        for tw in (64, 100, 211):
            scale, _, _ = vb.thumbnail_webp_scale(211, 150, tw)
            dec = vb.Image(vb.webp_decode_host_twin(s, scale=scale))
            want = dec.thumbnail_image(tw, output_profile=srgb, embedded_profile=prof, builtin_profiles=builtin).numpy()
            assert np.array_equal(vb.thumbnail_buffer(s, tw, output_profile=srgb, builtin_profiles=builtin), want), tw
            want = dec.thumbnail_image_linear(tw, output_profile=srgb, embedded_profile=prof, builtin_profiles=builtin).numpy()
            assert np.array_equal(vb.thumbnail_buffer_linear(s, tw, output_profile=srgb, builtin_profiles=builtin), want), tw


@pytest.mark.gpu
def test_gpu_plan_run_webp(vb):
    streams = [pil_webp(content("photo", 300, 400, 30 + i), quality=50 + 5 * i) for i in range(6)]
    streams += [vp8_stream(9200 + i, h=300, w=400) for i in range(4)]
    scale, sw, sh = vb.thumbnail_webp_scale(400, 300, 96)
    plan = vb.ThumbnailPlan(sw, sh, 3, 96)
    got = plan.run_webp(streams, scale)
    for i, s in enumerate(streams):
        assert np.array_equal(got[i], vb.thumbnail_buffer(s, 96)), i

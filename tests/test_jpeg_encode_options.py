"""vips_jpegsave's entropy-coding options on the device encoder (csrc/jpeg_encode.cu): optimize_coding
(jpegsave.c:227-232 -> vips2jpeg.c:590-591) and restart_interval (jpegsave.c:284-289 -> vips2jpeg.c:593-597).

Both change only libjpeg's entropy coder, so the oracle is the one the default path is held to: libjpeg-turbo inside this
image's Pillow (optimize=True, restart_marker_blocks=R), the whole stream byte for byte.  The table generator is also held
to libjpeg-turbo's own jpeg_gen_optimal_table, called through ctypes on Pillow's bundled libjpeg.

CPU tests run the host twin (vb200_debug_jpeg_encode_opts); -m gpu tests the kernels (vb200_jpegsave_batch_opts).
"""
import ctypes as C
import glob
import io
import os

import numpy as np
import pytest

PIL = pytest.importorskip("PIL.Image")

from test_jpeg import synth  # noqa: E402
from test_jpeg_encode import same_stream, segments  # noqa: E402

MODES = {"auto": 0, "on": 1, "off": 2}


def pil_sub(mode, q):
    return {"auto": 2 if q < 90 else 0, "on": 2, "off": 0}[mode]


def turbo(a, q, mode="auto", optimize=False, restart=0):
    b = io.BytesIO()
    kw = {}
    if optimize:
        kw["optimize"] = True
    if restart:
        kw["restart_marker_blocks"] = restart
    # vips2jpeg.c:678-684: one band is always 1 x 1
    PIL.fromarray(a).save(b, "JPEG", quality=q, subsampling=pil_sub(mode, q) if a.ndim == 3 else 0, **kw)
    return b.getvalue()


def mcu_count(a, q, mode):
    h, w = a.shape[:2]
    sub = a.ndim == 3 and pil_sub(mode, q) == 2
    m = 16 if sub else 8
    return ((w + m - 1) // m) * ((h + m - 1) // m)


def restarts(mcus):
    return sorted({0, 1, 2, 7, max(1, mcus - 1), mcus, mcus + 1, 65535})


def check(ours, theirs, what, restart):
    same_stream(ours, theirs, what)
    so, _ = segments(ours)
    if restart:
        assert so[0xDD] == [bytes([restart >> 8, restart & 255])], what
    else:
        assert 0xDD not in so, what


@pytest.fixture(scope="module")
def vb():
    import libvips_b200
    return libvips_b200


@pytest.fixture(scope="module")
def enc(vb):
    L = vb.lib()

    def run(a, q, mode="auto", optimize=False, restart=0):
        a = np.ascontiguousarray(a)
        h, w = a.shape[:2]
        bands = 1 if a.ndim == 2 else a.shape[2]
        cap = w * h * 8 + 3 * h * w // 16 + 8192
        buf = (C.c_ubyte * cap)()
        n = C.c_size_t()
        opts = vb.JpegSaveOptions(q, MODES[mode], int(optimize), restart)
        vb._check(L.vb200_debug_jpeg_encode_opts(a.ctypes.data_as(C.c_void_p), w * bands, w, h, bands, C.byref(opts), buf, cap, C.byref(n)))
        return bytes(buf[:n.value])
    return run


# ------------------------------------------------------------------ the table generator against libjpeg-turbo's own


class JHUFF_TBL(C.Structure):
    _fields_ = [("bits", C.c_ubyte * 17), ("huffval", C.c_ubyte * 256), ("sent_table", C.c_int)]


@pytest.fixture(scope="module")
def gen_pair(vb):
    libs = glob.glob(os.path.join(os.path.dirname(PIL.__file__), "..", "pillow.libs", "libjpeg*.so*"))
    fn = None
    for p in libs:
        try:
            fn = getattr(C.CDLL(p), "jpeg_gen_optimal_table")
            break
        except (OSError, AttributeError):
            pass
    if fn is None:
        pytest.skip("Pillow's libjpeg does not export jpeg_gen_optimal_table")
    fn.argtypes = [C.c_void_p, C.POINTER(JHUFF_TBL), C.POINTER(C.c_long)]
    fn.restype = None
    cinfo = C.create_string_buffer(8192)     # only read on an error exit, which these counts never reach
    L = vb.lib()

    def turbo_gen(freq):
        f = (C.c_long * 257)(*[int(v) for v in freq], 0)
        t = JHUFF_TBL()
        fn(cinfo, C.byref(t), f)
        n = sum(t.bits[1:])
        return list(t.bits), list(t.huffval[:n])

    def our_gen(freq):
        f = np.ascontiguousarray(freq, np.uint32)
        bits = (C.c_ubyte * 17)()
        hv = (C.c_ubyte * 256)()
        vb._check(L.vb200_debug_jpeg_optimal_table(f.ctypes.data_as(C.c_void_p), bits, hv))
        n = sum(bits[1:])
        return list(bits), list(hv[:n])
    return our_gen, turbo_gen


def test_generator_matches_libjpeg_turbo(gen_pair):
    ours, theirs = gen_pair
    vecs = []
    fib = [1, 1]
    while len(fib) < 30:
        fib.append(fib[-1] + fib[-2])
    f = np.zeros(256, np.int64)
    f[:30] = fib
    vecs.append(("fibonacci", f.copy()))
    f = np.zeros(256, np.int64)
    f[::-1][:30] = fib                               # the long codes on the high symbols
    vecs.append(("fibonacci reversed", f.copy()))
    f = np.zeros(256, np.int64)
    f[17] = 5
    vecs.append(("one symbol", f))
    vecs.append(("256 equal", np.full(256, 7, np.int64)))
    vecs.append(("ties", np.array([1 + (i % 3) for i in range(256)], np.int64)))
    rng = np.random.default_rng(11)
    for k in range(1000):
        f = np.zeros(256, np.int64)
        nz = rng.integers(1, 257)
        idx = rng.choice(256, nz, replace=False)
        f[idx] = rng.integers(1, [2, 10, 1000, 100000][k % 4], nz)
        vecs.append(("random %d" % k, f))
    deep = 0
    for what, f in vecs:
        got, want = ours(f), theirs(f)
        assert got == want, what
        deep += got[0][16] > 0 and what.startswith("fib")
    assert deep, "the Fibonacci vectors did not reach the 16-bit limit"
    # after the limit, huffval is not in order of final code length: a restatement that re-sorts would differ here
    bits, hv = ours(vecs[0][1])
    f = vecs[0][1]
    by_final = sorted(hv, key=lambda s: (-f[s], s))
    assert hv != by_final or bits[16] == 0


def test_generator_refuses_counts_past_the_sentinel(vb):
    f = np.zeros(256, np.uint32)
    f[0] = 10 ** 9
    assert vb.lib().vb200_debug_jpeg_optimal_table(f.ctypes.data_as(C.c_void_p), (C.c_ubyte * 17)(), (C.c_ubyte * 256)()) == -1


# ------------------------------------------------------------------ whole streams against Pillow (host twin)


@pytest.mark.parametrize("size", [(3, 5), (8, 8), (17, 300), (67, 93), (129, 31), (512, 512)], ids=lambda s: "%dx%d" % s)
def test_host_twin_writes_libjpeg_turbos_stream(enc, size):
    h, w = size
    a = synth(h, w, seed=h + 7 * w)
    g = synth(h, w, seed=w, grey=True)
    for i, q in enumerate((1, 50, 75, 89, 90, 100)):
        r = (0, 7)[i % 2]
        check(enc(a, q, "auto", True, r), turbo(a, q, "auto", True, r), (size, q, "optimise", r), r)
    for img, q, mode in ((a, 75, "auto"), (a, 95, "on"), (a, 75, "off"), (g, 75, "auto")):
        for r in restarts(mcu_count(img, q, mode)):
            for opt in (False, True):
                check(enc(img, q, mode, opt, r), turbo(img, q, mode, opt, r), (size, q, mode, img.ndim, opt, r), r)


def test_extremes(enc):
    rng = np.random.default_rng(5)
    noise = rng.integers(0, 256, (96, 128, 3), dtype=np.uint8)
    yy, xx = np.mgrid[0:64, 0:80]
    checker = np.repeat((((yy + xx) % 2) * 255).astype(np.uint8)[..., None], 3, -1)
    flat = np.full((40, 56, 3), 255, np.uint8)
    for name, a in (("noise", noise), ("flat", flat), ("inverted flat", 255 - flat), ("checker", checker)):
        for q in (1, 75, 100):
            for opt, r in ((True, 0), (True, 1), (False, 3), (True, 5)):
                check(enc(a, q, "auto", opt, r), turbo(a, q, "auto", opt, r), (name, q, opt, r), r)


def test_padding_bytes_are_stuffed(enc):
    """an interval whose last bits are all ones pads to an FF byte, which is stuffed; the marker after it is not"""
    rng = np.random.default_rng(9)
    seen = 0
    for k in range(6):
        a = rng.integers(0, 256, (64, 64), dtype=np.uint8)
        for opt in (False, True):
            d = enc(a, 100, "auto", opt, 1)
            check(d, turbo(a, 100, "auto", opt, 1), (k, opt), 1)
            seen += sum(d[i:i + 3] == b"\xff\x00\xff" and 0xD0 <= d[i + 3] <= 0xD7 for i in range(len(d) - 3))
    assert seen > 0, "no padding byte came out as 0xFF"


def test_refusals(enc, vb):
    a = synth(16, 16, seed=1)
    for r in (-1, 65536, 2 ** 31 - 1):
        with pytest.raises(vb.Error, match="restart_interval"):
            enc(a, 75, "auto", True, r)


def test_round_trip_through_the_device_decoder_twin(enc, vb):
    """an optimised stream with restart markers reads back through the decoder's restart-interval path as libjpeg-turbo
    reads it (the decoder refuses a stream whose markers do not follow its DRI)"""
    for a, r in ((synth(120, 200, seed=8), 3), (synth(67, 93, seed=2, grey=True), 1)):
        d = enc(a, 85, "auto", True, r)
        assert 0xDD in segments(d)[0]
        got = vb.jpeg_decode_host_twin(d, 1)
        want = np.asarray(PIL.open(io.BytesIO(d)))
        assert np.array_equal(got.reshape(want.shape), want)


# ------------------------------------------------------------------ the device encoder


def gpu_save(vb, frames, q, mode="auto", optimize=False, restart=0, frames_dev=False, out_dev=False):
    """vb200_jpegsave_batch_opts with frames and streams in host or device memory -> list of bytes"""
    import torch
    frames = np.ascontiguousarray(frames)
    if frames.ndim == 3:
        frames = frames[..., None]
    n, h, w, bands = frames.shape
    stride = w * h * bands * 2 + 3 * w * h // 16 + 4096
    lens = (C.c_size_t * n)()
    opts = vb.JpegSaveOptions(q, MODES[mode], int(optimize), restart)
    if frames_dev:
        ft = torch.from_numpy(frames).cuda()
        src, sw = C.c_void_p(ft.data_ptr()), vb.DEVICE
    else:
        src, sw = frames.ctypes.data_as(C.c_void_p), vb.HOST
    if out_dev:
        ot = torch.empty((n, stride), dtype=torch.uint8, device="cuda")
        dst, dw = C.c_void_p(ot.data_ptr()), vb.DEVICE
    else:
        oh = np.empty((n, stride), np.uint8)
        dst, dw = oh.ctypes.data_as(C.c_void_p), vb.HOST
    vb._check(vb.lib().vb200_jpegsave_batch_opts(src, sw, w * bands, w * h * bands, n, w, h, bands, C.byref(opts), dst, dw, stride, lens))
    if out_dev:
        torch.cuda.synchronize()
        oh = ot.cpu().numpy()
    return [oh[i, :lens[i]].tobytes() for i in range(n)]


@pytest.mark.gpu
def test_gpu_batch_writes_libjpeg_turbos_streams(vb):
    vb.init(0)
    k = 0
    for (h, w) in ((3, 5), (8, 8), (17, 300), (67, 93), (129, 31), (512, 512)):
        frames = np.stack([synth(h, w, seed=i + h + w) for i in range(3)])
        grey = frames[..., 1].copy()
        for imgs, q, mode in ((frames, 75, "auto"), (frames, 95, "on"), (frames, 60, "off"), (grey, 80, "auto"), (frames, 100, "auto"),
                              (frames, 1, "auto")):
            for r in restarts(mcu_count(imgs[0], q, mode)):
                for opt in (False, True):
                    k += 1
                    got = gpu_save(vb, imgs, q, mode, opt, r, frames_dev=bool(k & 1), out_dev=bool(k & 2))
                    for i in range(3):
                        check(got[i], turbo(imgs[i], q, mode, opt, r), ((h, w), q, mode, imgs.ndim, opt, r, i), r)
    rng = np.random.default_rng(6)
    noise = rng.integers(0, 256, (2, 96, 128, 3), dtype=np.uint8)
    got = vb.jpegsave_batch(noise, 100, optimize_coding=True, restart_interval=1)
    for i in range(2):
        check(got[i], turbo(noise[i], 100, "auto", True, 1), ("noise", i), 1)
    with pytest.raises(vb.Error, match="restart_interval"):
        vb.jpegsave_batch(noise, 75, restart_interval=65536)


@pytest.mark.gpu
def test_gpu_mixed_batch_has_its_own_tables_per_frame(vb, enc):
    vb.init(0)
    h, w = 96, 128
    rng = np.random.default_rng(7)
    yy, xx = np.mgrid[0:h, 0:w]
    frames = np.stack([rng.integers(0, 256, (h, w, 3), dtype=np.uint8), np.full((h, w, 3), 40, np.uint8),
                       np.repeat((((yy // 3 + xx // 3) % 2) * 255).astype(np.uint8)[..., None], 3, -1), synth(h, w, seed=3)])
    for r in (0, 5):
        got = vb.jpegsave_batch(frames, 75, optimize_coding=True, restart_interval=r)
        dhts = [tuple(segments(d)[0][0xC4]) for d in got]
        assert len(set(dhts)) == len(frames), "the frames' tables should all differ"
        for i in range(len(frames)):
            single = vb.jpegsave_batch(frames[i:i + 1], 75, optimize_coding=True, restart_interval=r)[0]
            assert got[i] == single, (r, i)
            assert got[i] == enc(frames[i], 75, "auto", True, r), (r, i)
            check(got[i], turbo(frames[i], 75, "auto", True, r), (r, i), r)


@pytest.mark.gpu
def test_gpu_70001_frames_in_one_call(vb, enc):
    """past the grid's 65 535 frames and more than two chunks of per-frame tables"""
    vb.init(0)
    n = 70001
    rng = np.random.default_rng(8)
    base = synth(16, 16, seed=1).astype(np.int16)
    frames = np.clip(base[None] + rng.integers(-40, 41, (n, 1, 1, 3)) + rng.integers(-8, 9, (n, 16, 16, 3)), 0, 255).astype(np.uint8)
    got = vb.jpegsave_batch(frames, 75, optimize_coding=True, restart_interval=1)
    bad = [i for i in range(n) if got[i] != enc(frames[i], 75, "auto", True, 1)]
    assert not bad, "frames %s differ from the host twin" % bad[:10]
    for i in rng.choice(n, 50, replace=False):
        check(got[i], turbo(frames[i], 75, "auto", True, 1), int(i), 1)


@pytest.mark.gpu
def test_gpu_jpeg_in_optimised_jpeg_out(vb):
    """the thumbnail server's loop: JPEG streams -> device thumbnail -> optimised save with restart markers, read back
    by the device decoder through its restart-interval path"""
    import torch
    from oracle import pyoracle
    from test_jpeg import encode, turbo_decode
    vb.init(0)
    h, w, target = 1024, 1536, 256
    streams = [encode(synth(h, w, seed=i), 88, 2) for i in range(3)]
    shrink = vb.thumbnail_jpegshrink(w, h, target)
    dw, dh, bands = vb.jpeg_geometry(streams, shrink)
    plan = vb.ThumbnailPlan(dw, dh, bands, target)
    out = torch.empty((3, plan.out_height, plan.out_width, bands), dtype=torch.uint8, device="cuda")
    plan.run_jpeg(streams, shrink, out_ptr=out.data_ptr())
    torch.cuda.synchronize()
    r = (plan.out_width + 15) // 16          # one restart interval per MCU row
    got = vb.jpegsave_batch(None, 75, in_ptr=out.data_ptr(), shape=tuple(out.shape), optimize_coding=True, restart_interval=r)
    for i in range(3):
        thumb = pyoracle.thumbnail_image(turbo_decode(streams[i], shrink), target)
        check(got[i], turbo(thumb, 75, "auto", True, r), i, r)
    back = vb.jpeg_decode_batch(got)
    for i in range(3):
        want = np.asarray(PIL.open(io.BytesIO(got[i])))
        assert np.array_equal(np.asarray(back[i]).reshape(want.shape), want), i


@pytest.mark.gpu
def test_gpu_default_options_are_the_plain_call(vb):
    vb.init(0)
    frames = np.stack([synth(67, 93, seed=i) for i in range(4)])
    n, h, w, bands = frames.shape
    stride = w * h * bands * 2 + 4096
    L = vb.lib()

    def run(call):
        out = np.zeros((n, stride), np.uint8)
        lens = (C.c_size_t * n)()
        before = vb.launch_count()
        vb._check(call(out, lens))
        return [out[i, :lens[i]].tobytes() for i in range(n)], vb.launch_count() - before
    src = frames.ctypes.data_as(C.c_void_p)
    plain = run(lambda o, l: L.vb200_jpegsave_batch(src, vb.HOST, w * bands, w * h * bands, n, w, h, bands, 75, 0, o.ctypes.data_as(C.c_void_p),
                                                   vb.HOST, stride, l))
    opts = vb.JpegSaveOptions(75, 0, 0, 0)
    withopts = run(lambda o, l: L.vb200_jpegsave_batch_opts(src, vb.HOST, w * bands, w * h * bands, n, w, h, bands, C.byref(opts),
                                                           o.ctypes.data_as(C.c_void_p), vb.HOST, stride, l))
    assert plain == withopts
    assert plain[1] == 7
    for opt, r, launches in ((True, 0, 9), (False, 4, 8), (True, 4, 10)):
        before = vb.launch_count()
        vb.jpegsave_batch(frames, 75, optimize_coding=opt, restart_interval=r)
        assert vb.launch_count() - before == launches, (opt, r)

"""Progressive JPEG save on the device encoder (csrc/jpeg_encode.cu): vips_jpegsave's interlace (jpegsave.c:234-238 ->
vips2jpeg.c:670-673, jpeg_simple_progression).

The oracle is libjpeg-turbo inside this image's Pillow (progressive=True makes the same jpeg_simple_progression call), the
whole stream byte for byte: SOF2, 10 scans for YCbCr and 6 for greyscale, a DHT before every scan but the DC refinement,
one DRI before the first SOS with restart markers.  libjpeg forces optimize_coding on in progressive mode, so the option
changes nothing.

CPU tests run the host twin (vb200_debug_jpeg_encode_opts), a serial restatement of jcphuff.c; -m gpu tests the kernels
(vb200_jpegsave_batch_opts), whose run structure is resolved by a chain walk over per-block summaries.
"""
import ctypes as C
import io

import numpy as np
import pytest

PIL = pytest.importorskip("PIL.Image")

from test_jpeg import synth  # noqa: E402
from test_jpeg_encode_options import MODES, mcu_count, pil_sub, restarts  # noqa: E402

# jcparam.c jpeg_simple_progression: (components, Ss, Se, Ah, Al) per scan
SCRIPT_YCC = [((1, 2, 3), 0, 0, 0, 1), ((1,), 1, 5, 0, 2), ((3,), 1, 63, 0, 1), ((2,), 1, 63, 0, 1), ((1,), 6, 63, 0, 2),
              ((1,), 1, 63, 2, 1), ((1, 2, 3), 0, 0, 1, 0), ((3,), 1, 63, 1, 0), ((2,), 1, 63, 1, 0), ((1,), 1, 63, 1, 0)]
SCRIPT_GREY = [((1,), 0, 0, 0, 1), ((1,), 1, 5, 0, 2), ((1,), 6, 63, 0, 2), ((1,), 1, 63, 2, 1), ((1,), 0, 0, 1, 0), ((1,), 1, 63, 1, 0)]


def turbo(a, q, mode="auto", optimize=False, restart=0):
    b = io.BytesIO()
    kw = {"progressive": True}
    if optimize:
        kw["optimize"] = True
    if restart:
        kw["restart_marker_blocks"] = restart
    PIL.fromarray(a).save(b, "JPEG", quality=q, subsampling=pil_sub(mode, q) if a.ndim == 3 else 0, **kw)
    return b.getvalue()


def markers(d):
    """every marker segment of the stream in order, [(marker, payload)], the entropy-coded data skipped"""
    out, p = [], 2
    assert d[:2] == b"\xff\xd8"
    while True:
        assert d[p] == 0xFF, p
        m = d[p + 1]
        if m == 0xD9:
            assert p + 2 == len(d), "bytes after EOI"
            return out
        n = (d[p + 2] << 8) | d[p + 3]
        out.append((m, bytes(d[p + 4:p + 2 + n])))
        p += 2 + n
        if m == 0xDA:
            # scan data: up to the next marker that is neither a stuffed zero nor RSTn
            while not (d[p] == 0xFF and d[p + 1] != 0 and not 0xD0 <= d[p + 1] <= 0xD7):
                p += 1


def check(ours, theirs, what, restart, grey):
    if ours != theirs:
        n = next((i for i in range(min(len(ours), len(theirs))) if ours[i] != theirs[i]), min(len(ours), len(theirs)))
        raise AssertionError(("streams differ at byte %d of %d / %d" % (n, len(ours), len(theirs)), what))
    ms = markers(ours)
    kinds = [m for m, _ in ms]
    assert 0xC2 in kinds and 0xC0 not in kinds, what
    script = SCRIPT_GREY if grey else SCRIPT_YCC
    sos = [i for i, m in enumerate(kinds) if m == 0xDA]
    assert len(sos) == len(script), what
    prev = kinds.index(0xC2)
    for i, (comps, ss, se, ah, al) in zip(sos, script):
        p = ms[i][1]
        assert tuple(p[1:1 + 2 * p[0]:2]) == comps and (p[-3], p[-2], p[-1] >> 4, p[-1] & 15) == (ss, se, ah, al), what
        between = kinds[prev + 1:i]
        assert (0xC4 in between) == (not (ss == 0 and ah > 0)), (what, "DHT before scan", ss, ah)
        prev = i
    dri = [i for i, m in enumerate(kinds) if m == 0xDD]
    if restart:
        assert len(dri) == 1 and dri[0] < sos[0] and ms[dri[0]][1] == bytes([restart >> 8, restart & 255]), what
    else:
        assert not dri, what


def unit_restarts(a, q, mode):
    """restart intervals around the unit counts of the single-component scans too (the luma block grid)"""
    h, w = a.shape[:2]
    luma = ((w + 7) // 8) * ((h + 7) // 8)
    return sorted(set(restarts(mcu_count(a, q, mode))) | {luma - 1, luma, luma + 1} - {0} | {0})


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
        cap = w * h * 8 + 3 * h * w // 16 + 16384
        buf = (C.c_ubyte * cap)()
        n = C.c_size_t()
        opts = vb.JpegSaveOptions(q, MODES[mode], int(optimize), restart, 1)
        vb._check(L.vb200_debug_jpeg_encode_opts(a.ctypes.data_as(C.c_void_p), w * bands, w, h, bands, C.byref(opts), buf, cap, C.byref(n)))
        return bytes(buf[:n.value])
    return run


@pytest.fixture(scope="module")
def events(vb):
    L = vb.lib()

    def run(a, q, mode="auto", restart=0):
        a = np.ascontiguousarray(a)
        h, w = a.shape[:2]
        bands = 1 if a.ndim == 2 else a.shape[2]
        e = (C.c_ulonglong * 3)()
        opts = vb.JpegSaveOptions(q, MODES[mode], 0, restart, 1)
        vb._check(L.vb200_debug_jpeg_prog_events(a.ctypes.data_as(C.c_void_p), w * bands, w, h, bands, C.byref(opts), e))
        return {"eob_7fff": e[0], "be_flush": e[1], "refine_zrl": e[2]}
    return run


# ------------------------------------------------------------------ the host twin against Pillow


SIZES = [(3, 5), (8, 8), (17, 300), (67, 93), (129, 31), (33, 47), (512, 512)]


@pytest.mark.parametrize("size", SIZES, ids=lambda s: "%dx%d" % s)
def test_host_twin_writes_libjpeg_turbos_progressive_stream(enc, size):
    """33 x 47 and 67 x 93 at 4:2:0: the luma grid is not a multiple of the MCU, so the luma scans skip dummy blocks"""
    h, w = size
    a = synth(h, w, seed=h + 7 * w)
    g = synth(h, w, seed=w, grey=True)
    for i, q in enumerate((1, 50, 75, 89, 90, 100)):
        r = (0, 7)[i % 2]
        check(enc(a, q, "auto", False, r), turbo(a, q, "auto", False, r), (size, q, r), r, False)
    for img, q, mode in ((a, 75, "auto"), (a, 95, "on"), (a, 75, "off"), (g, 75, "auto")):
        for r in unit_restarts(img, q, mode):
            ours = enc(img, q, mode, False, r)
            check(ours, turbo(img, q, mode, False, r), (size, q, mode, img.ndim, r), r, img.ndim == 2)
            # libjpeg forces optimize_coding on in progressive mode: the option changes no byte, here or in Pillow
            assert enc(img, q, mode, True, r) == ours, (size, q, mode, r)
            assert turbo(img, q, mode, True, r) == ours, (size, q, mode, r)


def test_eob_run_reaches_0x7fff(enc, events):
    """a flat 2048 x 1024 frame at Q 1: every AC block ends in an EOB, 32 768 of them per scan, so runs are forced out at
    0x7FFF blocks"""
    a = np.full((1024, 2048), 128, np.uint8)
    assert events(a, 1)["eob_7fff"] > 0
    check(enc(a, 1), turbo(a, 1), "flat", 0, True)
    rgb = np.full((1024, 2048, 3), (30, 140, 220), np.uint8)
    check(enc(rgb, 1, "off"), turbo(rgb, 1, "off"), "flat rgb", 0, False)


def test_correction_bits_flush_the_run(enc, events):
    """a checkerboard at Q 100: refinement blocks carry many correction bits and no newly non-zero coefficient, so the
    run is forced out once more than MAX_CORR_BITS - 63 bits are buffered"""
    yy, xx = np.mgrid[0:256, 0:256]
    a = (((yy + xx) % 2) * 255).astype(np.uint8)
    assert events(a, 100)["be_flush"] > 0
    for r in (0, 5, 40):
        check(enc(a, 100, "auto", False, r), turbo(a, 100, "auto", False, r), ("checker", r), r, True)
    rgb = np.stack([a, 255 - a, a], -1)
    assert events(rgb, 100)["be_flush"] > 0
    check(enc(rgb, 100), turbo(rgb, 100), "checker rgb", 0, False)


def test_zrl_inside_refinement_scans(enc, events):
    for a, q in ((synth(512, 512, seed=1), 75), (synth(300, 200, seed=4, grey=True), 90)):
        assert events(a, q)["refine_zrl"] > 0
        for r in (0, 3):
            check(enc(a, q, "auto", False, r), turbo(a, q, "auto", False, r), (a.shape, q, r), r, a.ndim == 2)


def test_noise_at_q100(enc):
    rng = np.random.default_rng(5)
    for a in (rng.integers(0, 256, (96, 128, 3), dtype=np.uint8), rng.integers(0, 256, (77, 61), dtype=np.uint8)):
        for mode in ("auto", "on"):
            for r in (0, 1, 5):
                check(enc(a, 100, mode, False, r), turbo(a, 100, mode, False, r), (a.shape, mode, r), r, a.ndim == 2)


def test_padding_ff_bytes_are_stuffed(enc):
    """a segment whose last bits are all ones pads to an FF byte, which is stuffed, at an interval end (then RSTn) and at
    a scan end (then the next scan's DHT or SOS, or EOI); the marker after it is not"""
    rng = np.random.default_rng(9)
    seen_rst = seen_scan = 0
    for k in range(40):
        a = rng.integers(0, 256, (32, 48), dtype=np.uint8)
        for r in (1, 3):
            d = enc(a, 100, "auto", False, r)
            check(d, turbo(a, 100, "auto", False, r), (k, r), r, True)
            for i in range(len(d) - 3):
                if d[i:i + 3] == b"\xff\x00\xff":
                    seen_rst += 0xD0 <= d[i + 3] <= 0xD7
                    seen_scan += d[i + 3] in (0xC4, 0xDA, 0xD9)
        if seen_rst and seen_scan:
            break
    assert seen_rst > 0, "no interval ended in an FF byte"
    assert seen_scan > 0, "no scan ended in an FF byte"


def test_refusals(enc, vb):
    a = synth(16, 16, seed=1)
    for r in (-1, 65536):
        with pytest.raises(vb.Error, match="restart_interval"):
            enc(a, 75, "auto", False, r)


def test_round_trip_through_the_decoder_twin(enc, vb):
    for a, r in ((synth(120, 200, seed=8), 0), (synth(120, 200, seed=8), 3), (synth(67, 93, seed=2, grey=True), 1)):
        d = enc(a, 85, "auto", False, r)
        got = vb.jpeg_decode_host_twin(d, 1)
        want = np.asarray(PIL.open(io.BytesIO(d)))
        assert np.array_equal(got.reshape(want.shape), want)


# ------------------------------------------------------------------ the device encoder


def gpu_save(vb, frames, q, mode="auto", optimize=False, restart=0, frames_dev=False, out_dev=False, interlace=True):
    """vb200_jpegsave_batch_opts with frames and streams in host or device memory -> list of bytes"""
    import torch
    frames = np.ascontiguousarray(frames)
    if frames.ndim == 3:
        frames = frames[..., None]
    n, h, w, bands = frames.shape
    stride = w * h * bands * 2 + 3 * w * h // 16 + 8192
    lens = (C.c_size_t * n)()
    opts = vb.JpegSaveOptions(q, MODES[mode], int(optimize), restart, int(interlace))
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
def test_gpu_batch_writes_libjpeg_turbos_progressive_streams(vb, enc):
    vb.init(0)
    k = 0
    for (h, w) in SIZES:
        frames = np.stack([synth(h, w, seed=i + h + w) for i in range(3)])
        grey = frames[..., 1].copy()
        for imgs, q, mode in ((frames, 75, "auto"), (frames, 95, "on"), (frames, 60, "off"), (grey, 80, "auto"), (frames, 100, "auto"),
                              (frames, 1, "auto"), (frames, 50, "auto"), (frames, 89, "auto"), (frames, 90, "auto")):
            for r in unit_restarts(imgs[0], q, mode):
                k += 1
                opt = bool(k & 4)
                got = gpu_save(vb, imgs, q, mode, opt, r, frames_dev=bool(k & 1), out_dev=bool(k & 2))
                for i in range(3):
                    check(got[i], turbo(imgs[i], q, mode, False, r), ((h, w), q, mode, imgs.ndim, opt, r, i), r, imgs.ndim == 3)
    rng = np.random.default_rng(6)
    noise = rng.integers(0, 256, (2, 96, 128, 3), dtype=np.uint8)
    yy, xx = np.mgrid[0:256, 0:256]
    checker = np.stack([(((yy + xx) % 2) * 255).astype(np.uint8)] * 2)
    flat = np.full((1, 1024, 2048), 128, np.uint8)
    for imgs, q, r in ((noise, 100, 1), (noise, 100, 0), (checker, 100, 0), (checker, 100, 5), (flat, 1, 0), (flat, 1, 7)):
        got = vb.jpegsave_batch(imgs, q, restart_interval=r, interlace=True)
        for i in range(len(imgs)):
            check(got[i], turbo(imgs[i], q, "auto", False, r), (imgs.shape, q, r, i), r, imgs.ndim == 3)
    with pytest.raises(vb.Error, match="restart_interval"):
        vb.jpegsave_batch(noise, 75, restart_interval=65536, interlace=True)


@pytest.mark.gpu
def test_gpu_mixed_batch_has_its_own_tables_per_frame(vb, enc):
    vb.init(0)
    h, w = 96, 128
    rng = np.random.default_rng(7)
    yy, xx = np.mgrid[0:h, 0:w]
    frames = np.stack([rng.integers(0, 256, (h, w, 3), dtype=np.uint8), np.full((h, w, 3), 40, np.uint8),
                       np.repeat((((yy // 3 + xx // 3) % 2) * 255).astype(np.uint8)[..., None], 3, -1), synth(h, w, seed=3)])
    for r in (0, 5):
        got = vb.jpegsave_batch(frames, 75, restart_interval=r, interlace=True)
        dhts = [tuple(p for m, p in markers(d) if m == 0xC4) for d in got]
        assert len(set(dhts)) == len(frames), "the frames' tables should all differ"
        for i in range(len(frames)):
            single = vb.jpegsave_batch(frames[i:i + 1], 75, restart_interval=r, interlace=True)[0]
            assert got[i] == single, (r, i)
            assert got[i] == enc(frames[i], 75, "auto", False, r), (r, i)
            check(got[i], turbo(frames[i], 75, "auto", False, r), (r, i), r, False)


@pytest.mark.gpu
def test_gpu_70001_frames_in_one_call(vb, enc):
    """past the grid's 65 535 frames and more than two chunks of per-frame tables"""
    vb.init(0)
    n = 70001
    rng = np.random.default_rng(8)
    base = synth(16, 16, seed=1).astype(np.int16)
    frames = np.clip(base[None] + rng.integers(-40, 41, (n, 1, 1, 3)) + rng.integers(-8, 9, (n, 16, 16, 3)), 0, 255).astype(np.uint8)
    got = vb.jpegsave_batch(frames, 75, restart_interval=1, interlace=True)
    bad = [i for i in range(n) if got[i] != enc(frames[i], 75, "auto", False, 1)]
    assert not bad, "frames %s differ from the host twin" % bad[:10]
    for i in rng.choice(n, 50, replace=False):
        check(got[i], turbo(frames[i], 75, "auto", False, 1), int(i), 1, False)


@pytest.mark.gpu
def test_gpu_jpeg_in_progressive_jpeg_out(vb):
    """the thumbnail server's loop: JPEG streams -> device thumbnail -> progressive save with restart markers, read back
    by the device decoder's progressive path"""
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
    r = (plan.out_width + 15) // 16          # one MCU row of the interleaved scans
    got = vb.jpegsave_batch(None, 75, in_ptr=out.data_ptr(), shape=tuple(out.shape), restart_interval=r, interlace=True)
    for i in range(3):
        thumb = pyoracle.thumbnail_image(turbo_decode(streams[i], shrink), target)
        check(got[i], turbo(thumb, 75, "auto", False, r), i, r, False)
    back = vb.jpeg_decode_batch(got)
    for i in range(3):
        want = np.asarray(PIL.open(io.BytesIO(got[i])))
        assert np.array_equal(np.asarray(back[i]).reshape(want.shape), want), i


@pytest.mark.gpu
def test_gpu_launch_counts(vb):
    """11 launches per chunk for a progressive save whatever the frame count and restart interval; the baseline paths
    keep 7 / 8 / 9 / 10"""
    vb.init(0)
    frames = np.stack([synth(67, 93, seed=i) for i in range(4)])
    for n in (1, 4):
        for r in (0, 1, 4):
            for opt in (False, True):
                before = vb.launch_count()
                vb.jpegsave_batch(frames[:n], 75, optimize_coding=opt, restart_interval=r, interlace=True)
                assert vb.launch_count() - before == 11, (n, r, opt)
    for opt, r, launches in ((False, 0, 7), (True, 0, 9), (False, 4, 8), (True, 4, 10)):
        before = vb.launch_count()
        vb.jpegsave_batch(frames, 75, optimize_coding=opt, restart_interval=r)
        assert vb.launch_count() - before == launches, (opt, r)

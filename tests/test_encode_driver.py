"""The encoders' shared driver (csrc/encode.cu): vb200_jpegsave_batch_opts and vb200_pngsave_batch check their arguments
alike before any device call, run in chunks bounded by the device budget, fail a stream longer than its slot before its
chunk writes anything, and place streams for the host only once every chunk has succeeded."""
import ctypes as C

import numpy as np
import pytest

import libvips_b200 as vb

W, H, BANDS = 40, 24, 3


def _err():
    e = vb.lib().vb200_error_buffer().decode()
    vb.lib().vb200_error_clear()
    return e


def _jpeg(frames, bpl, stride, n, out, lens, restart=0, where=vb.HOST, out_where=vb.HOST, slot=1 << 16, opts=True):
    o = vb.JpegSaveOptions(75, 0, 0, restart, 0)
    return vb.lib().vb200_jpegsave_batch_opts(frames, where, bpl, stride, n, W, H, BANDS, C.byref(o) if opts else None, out, out_where, slot, lens)


def _png(frames, bpl, stride, n, out, lens, level=6, where=vb.HOST, out_where=vb.HOST, slot=1 << 16, opts=True):
    o = vb.PngSaveOptions(level, 0, 1.0)
    return vb.lib().vb200_pngsave_batch(frames, where, bpl, stride, n, W, H, BANDS, C.byref(o) if opts else None, None, 0, out, out_where, slot,
                                        lens)


@pytest.mark.parametrize("save", [_jpeg, _png], ids=["jpeg", "png"])
def test_argument_errors_come_before_the_device(save):
    """the same refusals from both entry points, every one before the library touches a device (at the parent commit the
    JPEG stride checks came after ensure_init, so on a machine without a GPU they reported the missing device instead)"""
    frames = np.zeros((2, H, W, BANDS), np.uint8)
    src = frames.ctypes.data_as(C.c_void_p)
    out = np.zeros((2, 1 << 16), np.uint8)
    dst = out.ctypes.data_as(C.c_void_p)
    lens = (C.c_size_t * 2)()
    line = W * BANDS
    cases = [
        ((None, line, line * H, 2, dst, lens), {}, "null argument"),
        ((src, line, line * H, 2, None, lens), {}, "null argument"),
        ((src, line, line * H, 2, dst, lens), {"opts": False}, "null argument"),
        ((src, line, line * H, 0, dst, lens), {}, "null argument"),
        ((src, line - 1, line * H, 2, dst, lens), {}, "frame strides too small for 40 x 24 x 3"),
        ((src, line, line * H - 1, 2, dst, lens), {}, "frame strides too small for 40 x 24 x 3"),
    ]
    for args, kw, want in cases:
        assert save(*args, **kw) == -1
        assert want in _err(), (args, kw)
    # an option the encoder refuses, with lengths left null (PNG took no null lengths at the parent commit)
    bad = {"restart": 65536} if save is _jpeg else {"level": 3}
    assert save(src, line, line * H, 2, dst, None, **bad) == -1
    assert ("restart_interval 65536" if save is _jpeg else "compression 3 is not built") in _err()
    assert (out == 0).all()


def _synth(n, seed=0):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W]
    base = np.stack([(x * 5 + y * 3) % 256, (x * y) % 256, (255 - x * 4) % 256], -1)
    return np.stack([(base + rng.integers(0, 40, base.shape)) % 256 for _ in range(n)]).astype(np.uint8)


def _twin(a, opts):
    cap = 1 << 20
    buf = (C.c_ubyte * cap)()
    n = C.c_size_t()
    vb._check(vb.lib().vb200_debug_jpeg_encode_opts(np.ascontiguousarray(a).ctypes.data_as(C.c_void_p), W * BANDS, W, H, BANDS, C.byref(opts), buf,
                                                    cap, C.byref(n)))
    return bytes(buf[:n.value])


MODES = {"baseline": ((0, 0, 0), 7), "restart": ((0, 2, 0), 8), "optimize": ((1, 0, 0), 9), "both": ((1, 2, 0), 10),
         "interlace": ((0, 0, 1), 11)}


@pytest.mark.gpu
@pytest.mark.parametrize("mode", sorted(MODES))
def test_gpu_chunked_jpeg_matches_unchunked(mode):
    """JPEG save under a budget of one frame per chunk and under one of a few: every stream equals the host twin, from host
    and device frames with padded strides into host and device slots, and each chunk runs the mode's launches"""
    import torch
    vb.init(0)
    L = vb.lib()
    (opt, restart, interlace), per_chunk = MODES[mode]
    opts = vb.JpegSaveOptions(75, 0, opt, restart, interlace)
    n, line = 7, W * BANDS
    frames = _synth(n, seed=len(mode))
    want = [_twin(frames[i], opts) for i in range(n)]
    bpl, stride, slot = line + 13, (line + 13) * H + 7, 1 << 14
    padded = np.zeros((n * stride,), np.uint8)
    for i in range(n):
        padded[i * stride:i * stride + bpl * H].reshape(H, bpl)[:, :line] = frames[i].reshape(H, line)
    dev_in = torch.from_numpy(padded).cuda()
    unchunked = None
    for budget in (0, 1, 3 * 1024 * 1024):
        L.vb200_debug_png_set_budget(budget)
        try:
            for frames_dev in (False, True):
                for out_dev in (False, True):
                    src = C.c_void_p(dev_in.data_ptr()) if frames_dev else padded.ctypes.data_as(C.c_void_p)
                    out_t = torch.full((n, slot), 0xA5, dtype=torch.uint8, device="cuda")
                    out_h = np.full((n, slot), 0xA5, np.uint8)
                    dst = C.c_void_p(out_t.data_ptr()) if out_dev else out_h.ctypes.data_as(C.c_void_p)
                    lens = (C.c_size_t * n)()
                    before = vb.launch_count()
                    vb._check(L.vb200_jpegsave_batch_opts(src, vb.DEVICE if frames_dev else vb.HOST, bpl, stride, n, W, H, BANDS, C.byref(opts), dst,
                                                          vb.DEVICE if out_dev else vb.HOST, slot, lens))
                    launches = vb.launch_count() - before
                    got = out_t.cpu().numpy() if out_dev else out_h
                    what = (mode, budget, frames_dev, out_dev)
                    assert [got[i, :lens[i]].tobytes() for i in range(n)] == want, what
                    assert launches % per_chunk == 0, what
                    chunks = launches // per_chunk
                    if budget == 1:
                        assert chunks == n, what
                    elif budget == 0:
                        assert chunks == 1, what
                        unchunked = launches
                    else:
                        assert 1 <= chunks <= n, what
        finally:
            L.vb200_debug_png_set_budget(0)
    assert unchunked == per_chunk


@pytest.mark.gpu
@pytest.mark.parametrize("out_dev", [False, True], ids=["host_out", "device_out"])
def test_gpu_jpeg_overflow_writes_nothing(out_dev):
    """a 2-frame batch whose second stream overflows its slot fails naming frame 1, writes no slot (at the parent commit
    the device slots of the frames that fit were written), and leaves nothing allocated"""
    import torch
    vb.init(0)
    L = vb.lib()
    L.vb200_debug_dz_pool_used.restype = C.c_size_t
    opts = vb.JpegSaveOptions(75, 0, 0, 0, 0)
    frames = np.stack([np.zeros((H, W, BANDS), np.uint8), np.random.default_rng(5).integers(0, 256, (H, W, BANDS), dtype=np.uint8)])
    slot = len(_twin(frames[0], opts)) + 10
    assert len(_twin(frames[1], opts)) > slot
    vb.jpegsave_batch(frames, 75)
    pool = L.vb200_debug_dz_pool_used()
    out_t = torch.full((2, slot), 0xA5, dtype=torch.uint8, device="cuda")
    out_h = np.full((2, slot), 0xA5, np.uint8)
    dst = C.c_void_p(out_t.data_ptr()) if out_dev else out_h.ctypes.data_as(C.c_void_p)
    lens = (C.c_size_t * 2)()
    rc = L.vb200_jpegsave_batch_opts(frames.ctypes.data_as(C.c_void_p), vb.HOST, W * BANDS, W * H * BANDS, 2, W, H, BANDS, C.byref(opts), dst,
                                     vb.DEVICE if out_dev else vb.HOST, slot, lens)
    err = _err()
    assert rc == -1 and "frame 1:" in err and "does not fit the %d-byte slot" % slot in err, err
    got = out_t.cpu().numpy() if out_dev else out_h
    assert (got == 0xA5).all()
    assert L.vb200_debug_dz_pool_used() == pool


@pytest.mark.gpu
def test_gpu_pngsave_buffer_matches_the_batch():
    """vb200_pngsave_buffer's stream, sized by the stream alone, is the batch's and the host twin's, for a frame whose
    worst-case bound is far above its stream"""
    vb.init(0)
    a = np.zeros((600, 500, 3), np.uint8)
    a[100:200, 50:300] = (10, 200, 30)
    got = vb.Image(a).pngsave_buffer(7)
    assert len(got) * 100 < vb._png_stride(500, 600, 3, None)
    assert got == vb.pngsave_batch(a[None], 7)[0] == vb.pngsave_host_twin(a, 7)


@pytest.mark.gpu
@pytest.mark.parametrize("jpeg", [{}, {"optimize_coding": True, "restart_interval": 3}, {"interlace": True}], ids=["baseline", "opt_restart",
                                                                                                               "interlace"])
def test_gpu_dzsave_matches_the_twin(jpeg):
    """dzsave's tiles through the driver's packed host output equal the host twin's, with the default batch budget and with
    batches of a few tiles"""
    vb.init(0)
    L = vb.lib()
    a = np.random.default_rng(6).integers(0, 256, (530, 700, 3), dtype=np.uint8)
    want = [t.bytes for t in vb.dzsave_host_twin(a, **jpeg).tiles]
    assert [t.bytes for t in vb.dzsave(a, **jpeg).tiles] == want
    try:
        L.vb200_debug_dz_set_budget(4 << 20)
        assert [t.bytes for t in vb.dzsave(a, **jpeg).tiles] == want
    finally:
        L.vb200_debug_dz_set_budget(0)

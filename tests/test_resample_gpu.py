"""GPU parity: the CUDA resample path (through the C ABI) against the CPU oracle.

Bit-exact for every integer format; float paths must be bit-identical too
(double accumulation in the same order, no FMA contraction) -- asserted as
max |diff| == 0, which is stricter than the 1 ULP the spec allows.

Structure follows the reference's test/test-suite/test_resample.py: every
format x kernel x factor, constant images, geometry/rounding, thumbnails.
"""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ALL_DTYPES = [np.uint8, np.int8, np.uint16, np.int16, np.uint32, np.int32, np.float32]
KERNELS = ["nearest", "linear", "cubic", "mitchell", "lanczos2", "lanczos3", "mks2013", "mks2021"]


def rand_image(rng, h, w, b, dt):
    dt = np.dtype(dt)
    if dt.kind == "f":
        return (rng.random((h, w, b), dtype=np.float32) * 255).astype(dt)
    info = np.iinfo(dt)
    return rng.integers(info.min, int(info.max) + 1, (h, w, b), dtype=np.int64).astype(dt)


def same(a, b):
    assert a.shape == b.shape, (a.shape, b.shape)
    assert a.dtype == b.dtype, (a.dtype, b.dtype)
    if not np.array_equal(a, b):
        d = np.abs(a.astype(np.float64) - b.astype(np.float64))
        idx = np.unravel_index(np.argmax(d), d.shape)
        raise AssertionError("max diff %g at %s (%s vs %s), %d differing" % (d.max(), idx, a[idx], b[idx], (d > 0).sum()))


@pytest.mark.parametrize("dt", ALL_DTYPES)
@pytest.mark.parametrize("bands", [1, 3, 4])
def test_shrink(vb, oracle, dt, bands):
    rng = np.random.default_rng(11)
    a = rand_image(rng, 67, 93, bands, dt)
    for f in (2, 3, 4, 7):
        for ceil in (False, True):
            same(vb.Image(a).shrinkv(f, ceil=ceil).numpy(), oracle.shrinkv(a, f, ceil))
            same(vb.Image(a).shrinkh(f, ceil=ceil).numpy(), oracle.shrinkh(a, f, ceil))


@pytest.mark.parametrize("dt", ALL_DTYPES)
@pytest.mark.parametrize("kernel", KERNELS)
def test_reduce_all_formats_kernels(vb, oracle, dt, kernel):
    """test_resample.py:77-92 shape: formats x kernels x factors."""
    rng = np.random.default_rng(5)
    a = rand_image(rng, 61, 83, 3, dt)
    for fac in (1.0, 1.1, 1.5, 1.999, 2.0, 3.3):
        v = vb.Image(a).reducev(fac, kernel=kernel).numpy()
        same(v, oracle.reducev(a, fac, kernel, 0.0, rect_h=16))
        h = vb.Image(a).reduceh(fac, kernel=kernel).numpy()
        same(h, oracle.reduceh(a, fac, kernel, 0.0, rect_w=0))


@pytest.mark.parametrize("kernel", KERNELS)
def test_constant_images_survive(vb, kernel):
    """test_resample.py:94-103: a constant uchar image reduced x2 stays constant."""
    for const in (0, 1, 2, 254, 255):
        a = np.full((10, 10, 1), const, np.uint8)
        r = vb.Image(a).reduce(2, 2, kernel=kernel).numpy()
        assert r.shape == (5, 5, 1)
        assert (r == const).all(), (kernel, const, r.ravel())


def test_reduce_gap(vb, oracle):
    rng = np.random.default_rng(7)
    a = rand_image(rng, 301, 257, 4, np.uint8)
    for fac in (4.0, 5.5, 8.0, 9.4):
        same(vb.Image(a).reducev(fac, gap=2.0).numpy(), oracle.reducev(a, fac, "lanczos3", 2.0, rect_h=128))
        same(vb.Image(a).reduceh(fac, gap=2.0).numpy(), oracle.reduceh(a, fac, "lanczos3", 2.0, rect_w=0))


def test_reduce_49_tap(vb, oracle):
    """BASELINE config 1 arithmetic (gap 0, shrink 8 => 49 taps) at a small size."""
    rng = np.random.default_rng(8)
    a = rand_image(rng, 512, 384, 4, np.uint8)
    v = vb.Image(a).reducev(8.0).numpy()
    same(v, oracle.reducev(a, 8.0, "lanczos3", 0.0, rect_h=16))
    same(vb.Image(v).reduceh(8.0).numpy(), oracle.reduceh(v, 8.0, "lanczos3", 0.0, rect_w=0))


@pytest.mark.parametrize("kernel", ["lanczos3", "lanczos2", "cubic", "linear", "nearest", "mks2021"])
def test_reduce_uchar_dp2a_kernels(vb, oracle, kernel):
    """The register-blocked IDP.2A leaf kernels (reducev_u8_dp2a_kernel: any band count with 4-byte rows,
    reduceh_u8x4_dp2a_kernel: RGBA): even / odd tap counts, factors whose per-rect stepping changes phase from
    tile to tile, windows hanging over both edges, images smaller than a row block / a CTA's span, row counts that
    are not a multiple of the block, and a tap count too large for their shared memory (falls back)."""
    rng = np.random.default_rng(11)
    for (h, w, b) in ((301, 260, 4), (67, 36, 4), (130, 512, 3), (5, 8, 4), (97, 1031, 4)):
        a = rand_image(rng, h, w, b, np.uint8)
        for fac in (1.0, 1.7, 2.0, 2.37, 3.3, 8.0, 13.0):
            if fac > min(h, w):
                continue
            same(vb.Image(a).reducev(fac, kernel=kernel).numpy(), oracle.reducev(a, fac, kernel, 0.0, rect_h=16))
            same(vb.Image(a).reduceh(fac, kernel=kernel).numpy(), oracle.reduceh(a, fac, kernel, 0.0, rect_w=0))
    a = rand_image(rng, 2100, 64, 4, np.uint8)
    same(vb.Image(a).reducev(49.0, kernel=kernel).numpy(), oracle.reducev(a, 49.0, kernel, 0.0, rect_h=16))
    a = rand_image(rng, 16, 2100, 4, np.uint8)
    same(vb.Image(a).reduceh(49.0, kernel=kernel).numpy(), oracle.reduceh(a, 49.0, kernel, 0.0, rect_w=0))
    # extremes that would overflow anything narrower than the reference's int sums
    for const in (0, 255):
        a = np.full((64, 64, 4), const, np.uint8)
        same(vb.Image(a).reduce(8.0, 8.0, kernel=kernel).numpy(), oracle.reduceh(oracle.reducev(a, 8.0, kernel, 0.0, rect_h=16), 8.0, kernel, 0.0, rect_w=0))


@pytest.mark.parametrize("dt", [np.uint8, np.uint16, np.int16, np.float32])
def test_premultiply_roundtrip_ops(vb, oracle, dt):
    rng = np.random.default_rng(3)
    for bands in (2, 4, 5):
        a = rand_image(rng, 33, 47, bands, dt)
        if np.dtype(dt).kind == "f":
            a[..., -1] = rng.random((33, 47), dtype=np.float32) * 300 - 20  # incl. out-of-range alpha
        ma = 255.0
        same(vb.Image(a).premultiply(max_alpha=ma).numpy(), oracle.premultiply(a, ma, False))
        same(vb.Image(a).unpremultiply(max_alpha=ma).numpy(), oracle.unpremultiply(a, ma, False))
        if dt == np.uint8:
            same(vb.Image(a).premultiply(uchar=True).numpy(), oracle.premultiply(a, 255.0, True))
            same(vb.Image(a).unpremultiply(uchar=True).numpy(), oracle.unpremultiply(a, 255.0, True))


def test_premultiply_all_alpha_values(vb, oracle):
    """every (value, alpha) pair through both uchar LUT paths"""
    v, al = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8))
    a = np.stack([v, v[::-1], v.T, al], axis=-1)
    same(vb.Image(a).premultiply(uchar=True).numpy(), oracle.premultiply(a, 255.0, True))
    same(vb.Image(a).unpremultiply(uchar=True).numpy(), oracle.unpremultiply(a, 255.0, True))


@pytest.mark.parametrize("dt", [np.uint8, np.uint16, np.float32])
def test_resize(vb, oracle, dt):
    """test_resample.py:113-146 geometry + parity"""
    rng = np.random.default_rng(21)
    a = rand_image(rng, 300, 401, 3, dt)
    for scale in (0.25, 0.5, 0.37, 0.11, 0.9):
        r = vb.Image(a).resize(scale).numpy()
        same(r, oracle.resize(a, scale))
    r = vb.Image(a).resize(0.3, vscale=0.7, kernel="cubic").numpy()
    same(r, oracle.resize(a, 0.3, 0.7, kernel="cubic"))
    # round-to-nearest sizing: 100x1 -> 50x1; 1600x1000 -> 10x6
    assert vb.Image(np.zeros((1, 100, 1), np.uint8)).resize(0.5).numpy().shape == (1, 50, 1)
    r = vb.Image(np.zeros((1000, 1600, 1), np.uint8)).resize(10.0 / 1600).numpy()
    assert r.shape[:2] == (6, 10)


def test_resize_edges_not_black(vb):
    """test_resample.py:131-146: no black edge pixels at /8, /9.4, /16"""
    a = np.full((600, 800, 3), 200, np.uint8)
    for scale in (1 / 8.0, 1 / 9.4, 1 / 16.0):
        r = vb.Image(a).resize(scale).numpy()
        assert r[0].min() > 190 and r[-1].min() > 190 and r[:, 0].min() > 190 and r[:, -1].min() > 190


def structured_rgba(h, w, kind, rng):
    a = np.zeros((h, w, 4), np.uint8)
    if kind == "random":
        a = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    elif kind.startswith("const"):
        a[...] = int(kind[5:])
    elif kind == "impulse":
        a[..., 3] = 255
        a[h // 2, w // 2] = 255
    elif kind == "hramp":
        a[...] = (np.arange(w) % 256).astype(np.uint8)[None, :, None]
    elif kind == "vramp":
        a[...] = (np.arange(h) % 256).astype(np.uint8)[:, None, None]
    elif kind.startswith("alpha"):
        a = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        a[..., 3] = int(kind[5:])
    return a


@pytest.mark.parametrize("kind", ["random", "const0", "const1", "const254", "const255", "impulse", "hramp", "vramp",
                                  "alpha0", "alpha1", "alpha128", "alpha255"])
def test_thumbnail_rgba_fused_structured(vb, oracle, kind):
    """SURVEY 8(d) structured cases through the fused kernel, 1024 -> 128 (shrink 8: the
    BASELINE chain premultiply/shrinkv4/reducev13/shrinkh4/reduceh13/unpremultiply)."""
    rng = np.random.default_rng(1234)
    a = structured_rgba(1024, 1024, kind, rng)
    plan = vb.ThumbnailPlan(1024, 1024, 4, 128)
    assert plan.fused
    same(plan.run_host(a[None])[0], oracle.thumbnail_image(a, 128))
    same(vb.Image(a).thumbnail_image(128).numpy(), oracle.thumbnail_image(a, 128))


@pytest.mark.parametrize("shape,target", [((997, 761), 100), ((761, 997), 100), ((640, 480), 64), ((300, 300), 150),
                                           ((1000, 1000), 143), ((2048, 1024), 300), ((333, 1999), 77)])
def test_thumbnail_rgba_odd_geometry(vb, oracle, shape, target):
    """fractional residual shrinks, non-multiple sizes, edges: fused vs oracle"""
    rng = np.random.default_rng(99)
    a = rng.integers(0, 256, shape + (4,), dtype=np.uint8)
    got = vb.Image(a).thumbnail_image(target).numpy()
    same(got, oracle.thumbnail_image(a, target))


@pytest.mark.parametrize("bands", [1, 2, 3])
def test_thumbnail_other_bands(vb, oracle, bands):
    rng = np.random.default_rng(17)
    a = rng.integers(0, 256, (700, 900, bands), dtype=np.uint8)
    same(vb.Image(a).thumbnail_image(120).numpy(), oracle.thumbnail_image(a, 120))


def test_thumbnail_force_and_down(vb, oracle):
    rng = np.random.default_rng(18)
    a = rng.integers(0, 256, (800, 1200, 4), dtype=np.uint8)
    same(vb.Image(a).thumbnail_image(100, 300, size="force").numpy(), oracle.thumbnail_image(a, 100, 300, "force"))
    same(vb.Image(a).thumbnail_image(200, size="down").numpy(), oracle.thumbnail_image(a, 200, size="down"))


def test_thumbnail_4k_full_size(vb, oracle):
    """BASELINE config 2 frame: 4096x4096 RGBA -> 512x512, bit-exact."""
    rng = np.random.default_rng(1234)
    a = rng.integers(0, 256, (4096, 4096, 4), dtype=np.uint8)
    same(vb.Image(a).thumbnail_image(512).numpy(), oracle.thumbnail_image(a, 512))


def test_thumbnail_avg_preserved(vb):
    """test_resample.py:171-205: thumbnail average within 1 of the source"""
    rng = np.random.default_rng(4)
    a = rng.integers(0, 256, (1000, 1500, 3), dtype=np.uint8)
    t = vb.Image(a).thumbnail_image(100)
    assert t.width == 100 and t.height == 67
    assert abs(t.avg() - a.mean()) < 1


def test_batch_device_and_pump(vb, oracle):
    """device-resident batch API (torch only holds the memory) and the host pump"""
    import torch
    rng = np.random.default_rng(1234)
    frames = rng.integers(0, 256, (5, 512, 768, 4), dtype=np.uint8)
    plan = vb.ThumbnailPlan(768, 512, 4, 96)
    want = np.stack([oracle.thumbnail_image(f, 96) for f in frames])
    din = torch.from_numpy(frames).cuda()
    dout = torch.zeros((5, plan.out_height, plan.out_width, 4), dtype=torch.uint8, device="cuda")
    vb.set_stream(torch.cuda.current_stream().cuda_stream)
    before = vb.launch_count()
    plan.run_device(din.data_ptr(), dout.data_ptr(), 5)
    torch.cuda.synchronize()
    vb.set_stream(0)
    assert vb.launch_count() > before
    same(dout.cpu().numpy(), want)
    same(plan.run_host(frames), want)


def test_tile_invariance_exact_shrinks(vb):
    """test/test_threading.sh invariant: output independent of tile geometry when
    the shrink is exactly representable (shrink 8 here)."""
    rng = np.random.default_rng(6)
    a = rng.integers(0, 256, (1024, 1024, 4), dtype=np.uint8)
    base = vb.Image(a).thumbnail_image(128).numpy()
    try:
        for tw, th in ((10, 10), (64, 64), (512, 512)):
            vb.set_tile_geometry(tw, th)
            same(vb.Image(a).thumbnail_image(128).numpy(), base)
    finally:
        vb.set_tile_geometry(128, 128, 16, 1)


def test_tile_geometry_changes_phase_tables(vb, oracle):
    """a non-representable shrink: results must follow the tile geometry the
    reference would have used (sequential X += shrink per rect)"""
    rng = np.random.default_rng(61)
    a = rng.integers(0, 256, (999, 1001, 4), dtype=np.uint8)
    try:
        for tw, th in ((64, 64), (128, 128)):
            vb.set_tile_geometry(tw, th)
            same(vb.Image(a).thumbnail_image(123).numpy(), oracle.thumbnail_image(a, 123, tile=(tw, th)))
    finally:
        vb.set_tile_geometry(128, 128, 16, 1)


V4_CASES = [
    # (W, H, target_w, target_h, size, has_alpha, frames, tensor-pipe kernel expected)
    (2048, 2048, 256, None, "both", True, 3, True),     # VS 4, HS 4: the headline's shape at 1/2 scale
    (1024, 1024, 256, None, "both", True, 2, True),     # 2, 2
    (1600, 1200, 200, None, "both", True, 1, True),     # 4, 4, one frame: rows split over CTAs
    (2048, 1024, 256, 256, "force", True, 2, True),     # V 2, H 4
    (1024, 2048, 256, 256, "force", True, 2, True),     # V 4, H 2
    (4096, 512, 256, 128, "force", True, 1, True),      # V 2, H 8
    (1600, 1600, 200, None, "both", False, 2, True),    # 4, 4 without alpha: no premultiply
    (4096, 4096, 512, None, "both", True, 2, True),     # the headline frame
    (2000, 1000, 420, None, "both", True, 2, True),     # residual 2.38, 15 taps: 5 output rows per chunk
    (3000, 2000, 640, None, "both", True, 1, True),     # shrink 4.69
    (4000, 3000, 410, None, "both", True, 1, True),     # shrink 9.76: box 4, residual 2.44
    (4096, 4096, 256, None, "both", True, 2, True),     # shrink 16: box 8 on both axes
    (3840, 2160, 225, None, "both", True, 1, True),     # shrink 17.07: box 8, residual 2.13
    # boxes that are not powers of two (multiplier-form averages, re-mapped fragment columns)
    (1200, 900, 150, None, "both", True, 1, True),      # V 3, H 4
    (3000, 2000, 428, None, "both", True, 2, True),     # 3, 3: shrink 7.01
    (2400, 1800, 340, None, "both", False, 1, True),    # 3, 3 without alpha
    (4000, 3000, 364, None, "both", True, 1, True),     # 5, 5: shrink 10.99
    (4096, 4096, 320, None, "both", True, 1, True),     # 6, 6: shrink 12.8
    (4096, 4096, 280, None, "both", True, 1, True),     # 7, 7: shrink 14.6
    (1920, 1080, 274, None, "both", True, 3, True),     # 3, 3 on a 16:9 frame, three frames
    (2048, 1536, 256, 256, "force", True, 1, True),     # V 3, H 4 in force mode
    (4096, 2048, 500, None, "both", True, 1, True),     # 4, 4 ... (shrink 8.19: box 4, residual 2.05)
    # plans the tensor-pipe kernel declines: rows not 16-byte aligned; boxes that differ by two.  They must land on
    # the older fused kernels with the same pixels
    (1003, 2057, 120, None, "both", True, 2, False),
    (2560, 1280, 256, 183, "force", True, 1, False),
    (2052, 2052, 128, None, "both", True, 1, False),     # box 8 whose last box runs past the frame's right edge
]


@pytest.mark.parametrize("case", V4_CASES, ids=lambda c: "%dx%d-%s" % (c[0], c[1], c[2]))
def test_thumbnail_tensor_pipe_kernel(vb, oracle, case):
    """The headline kernel (reducev as u8 x s8 MMAs, thumbnail_fused_mma.cuh) on every (VS, HS)
    corner it is instantiated for, batches of 1..3 frames, bit-exact against the oracle."""
    w, h, tw, th, size, alpha, n, mma = case
    rng = np.random.default_rng(w * 31 + h)
    frames = rng.integers(0, 256, (n, h, w, 4), dtype=np.uint8)
    frames[0, : h // 3, :, 3] = 255     # an opaque region and a transparent one
    frames[0, -(h // 5):, :, 3] = 0
    plan = vb.ThumbnailPlan(w, h, 4, tw, th, size=size, has_alpha=alpha)
    assert plan.fused, plan.kernel
    assert ("mma_kernel" in plan.kernel) == mma, plan.kernel
    want = np.stack([oracle.thumbnail_image(f, tw, th, size, has_alpha=alpha) for f in frames])
    same(plan.run_host(frames), want)


@pytest.mark.parametrize("shape", [(2048, 2048, 256), (1200, 900, 150), (4096, 4096, 256)], ids=lambda c: "%dx%d-%d" % c)
def test_thumbnail_opaque_stage_vote(vb, oracle, shape):
    """The tensor-pipe kernel's opaque fast path (a warp whose stage holds only alpha 255 skips the premultiply
    arithmetic; a warp that met live alpha probes every 8th stage): opaque frames, one stray pixel, alpha 254,
    opaque / live blocks finer and coarser than a warp's columns and a stage's rows, and the probe turned off."""
    w, h, tw = shape
    rng = np.random.default_rng(w + h)
    frames = rng.integers(0, 256, (6, h, w, 4), dtype=np.uint8)
    frames[0, :, :, 3] = 255                                 # opaque
    frames[1, :, :, 3] = 255
    frames[1, h // 2 + 3, w // 3 + 1, 3] = 17                # one live pixel in an opaque frame
    frames[2, :, :, 3] = 254                                 # nearly
    yy, xx = np.mgrid[0:h, 0:w]
    frames[3, :, :, 3] = np.where(((yy // 8) + (xx // 64)) % 2 == 0, 255, frames[3, :, :, 3])    # stage x warp checkerboard
    frames[4, :, :, 3] = np.where((yy // 97) % 3 != 1, 255, frames[4, :, :, 3])                  # long opaque / live runs of rows
    frames[5, :, :, 3] = np.where((xx // 5) % 7 == 0, frames[5, :, :, 3], 255)                   # live columns inside every warp
    plan = vb.ThumbnailPlan(w, h, 4, tw)
    assert "mma_kernel" in plan.kernel, plan.kernel
    want = np.stack([oracle.thumbnail_image(f, tw) for f in frames])
    # VB200_OPAQUE_PROBE: 2 = the voting instantiation from the first launch on, 0 = never, unset = a plan
    # switches to it once the hints of its earlier batches (read back asynchronously) found opaque frames
    for mode in ("2", "0", None):
        if mode is None:
            os.environ.pop("VB200_OPAQUE_PROBE", None)
        else:
            os.environ["VB200_OPAQUE_PROBE"] = mode
        try:
            for _ in range(3 if mode is None else 1):
                same(plan.run_host(frames), want)
                same(plan.run_host(frames[2:3]), want[2:3])     # a batch without a hinted frame in between
        finally:
            os.environ.pop("VB200_OPAQUE_PROBE", None)


@pytest.mark.parametrize("pad,shift", [(0, 0), (4096, 0), (48, 0), (20, 0), (0, 4)])
def test_batch_device_strides_and_alignment(vb, oracle, pad, shift):
    """Frame strides with padding (multiples of 16 keep the TMA kernels, others fall back to the
    ld.global kernel) and a base pointer off the 16-byte grid: same pixels on every path."""
    import torch
    rng = np.random.default_rng(77)
    n, h, w = 3, 512, 1024
    frame_bytes = h * w * 4
    stride = frame_bytes + pad
    raw = torch.zeros(shift + n * stride + 64, dtype=torch.uint8, device="cuda")
    frames = rng.integers(0, 256, (n, h, w, 4), dtype=np.uint8)
    for i in range(n):
        raw[shift + i * stride: shift + i * stride + frame_bytes] = torch.from_numpy(frames[i].reshape(-1)).cuda()
    plan = vb.ThumbnailPlan(w, h, 4, 128)
    out = torch.zeros((n, plan.out_height, plan.out_width, 4), dtype=torch.uint8, device="cuda")
    vb.set_stream(torch.cuda.current_stream().cuda_stream)
    L = vb.lib()
    L.vb200_thumbnail_batch_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]
    vb._check(L.vb200_thumbnail_batch_device(plan._p, raw.data_ptr() + shift, stride, out.data_ptr(),
                                             plan.out_frame_bytes, n))
    torch.cuda.synchronize()
    vb.set_stream(0)
    want = np.stack([oracle.thumbnail_image(f, 128) for f in frames])
    same(out.cpu().numpy(), want)


@pytest.mark.parametrize("shape,target", [((1024, 1024), 128), ((1200, 900), 150), ((600, 404), 99), ((2048, 1536), 256)])
def test_rgb_frames_ride_the_fused_rgba_kernels(vb, oracle, shape, target):
    """3-band 8-bit frames (what a JPEG decodes to): expanded to RGBX on the device, the fused RGBA kernel without
    premultiply, compacted -- the channels of the uchar chain never mix, so the bytes are the reference's"""
    from oracle import pyconv
    rng = np.random.default_rng(shape[0])
    h, w = shape
    frames = rng.integers(0, 256, (3, h, w, 3), dtype=np.uint8)
    plan = vb.ThumbnailPlan(w, h, 3, target)
    assert plan.fused, plan.kernel
    got = plan.run_host(frames)
    for i in range(3):
        assert np.array_equal(got[i], oracle.thumbnail_image(frames[i], target)), i
    assert np.array_equal(vb.Image(frames[0]).thumbnail_image(target).numpy(), got[0])
    plan.set_sharpen()
    got = plan.run_host(frames[:1])
    assert np.array_equal(got[0], pyconv.sharpen(oracle.thumbnail_image(frames[0], target), "srgb"))

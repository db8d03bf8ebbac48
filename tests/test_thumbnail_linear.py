"""linear=TRUE thumbnails (SURVEY 3.1b): sRGB -> scRGB, float premultiply / resize /
unpremultiply, scRGB -> sRGB.  Known answer from the reference's test-suite
(test_resample.py:234-238) + GPU parity against the oracle."""
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
FIX = np.load(os.path.join(HERE, "golden", "rgba_fixture.npz"))


def flatten_avg(t):
    t = t.astype(np.float64)
    al = t[..., 3:4] / 255.0
    return float((t[..., :3] * al + 255.0 * (1 - al)).mean())


def sweep_frame(h, w, bands, seed):
    """A frame for the kernel sweep: random bytes with every value 0 .. 255 in each channel (the first 256 pixels); RGBA
    frames then have an opaque quarter of rows, a transparent quarter and a last quarter whose alpha bytes step 1, 2, 3, 4
    across the width, so that reduced alpha falls on both sides of unpremultiply's |alpha| < 0.01 (2 / 255 and 3 / 255 lie
    either side of it)."""
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 256, (h, w, bands), dtype=np.uint8)
    flat = a.reshape(-1, bands)
    for c in range(bands):
        flat[:256, c] = rng.permutation(256)
    if bands == 4:
        q = h // 4
        a[q:2 * q, :, 3] = 255
        a[2 * q:3 * q, :, 3] = 0
        a[3 * q:, :, 3] = 1 + np.arange(w) * 4 // w
    return a


def v_form(w, h, bands, tw, th):
    """The kernel V a linear plan of vips_thumbnail(w x h, tw, th, size="force") launches, by linear_thumb_new's rule
    (libvips_b200/csrc/thumbnail_linear.cu): ("v2" for the residual-2.0 schedule linear_v2_kernel, else "v", bands, VST,
    whether the rows come through the cp.async ring).  The plan reduces by 1 / (1 / vshrink), as vips_resize does."""
    from oracle import pyoracle as orc
    _, vs, _, _ = orc.thumbnail_size(w, h, tw, th, "force")
    g = orc.reduce_geometry(h, 1.0 / max(1.0 / vs, 1.0 / h), "lanczos3", 2.0)
    vst = g.int_shrink if g.int_shrink in (2, 4, 8) else 0
    static2 = bands == 4 and vst != 0 and g.n_point == 13 and g.residual == 2.0
    return ("v2" if static2 else "v", bands, vst, bands == 4 and g.int_shrink <= 8)


def v_splits(w, oh, n, sm_count):
    """kernel V's row split for n frames: CTAs of one frame's column block share its output rows while the grid is
    small (linear_thumb_run, thumbnail_linear.cu), so splits > 1 starts CTAs at y_begin > 0"""
    col_blocks, splits = -(-w // 256), 1
    while col_blocks * splits * n < 4 * sm_count and oh // (splits * 2) >= 16:
        splits *= 2
    return splits


# (w, h, bands, target w, target h), size="force": the smallest frames that give each vertical shrink 32 output rows (so one
# frame splits its rows over CTAs), and horizontal shrinks of 5 to 7.5, most of them fractional.  A batch of 4 x SM-count / column
# blocks frames must fit the host pump's 64 MiB slice, so frames wider than 256 columns are short.
SWEEP = [
    (300, 128, 4, 40, 32),   # vshrink 4: box 2, residual 2.0 -> linear_v2_kernel<2>
    (61, 256, 4, 11, 32),    # vshrink 8: box 4 -> linear_v2_kernel<4>
    (53, 512, 4, 10, 32),    # vshrink 16: box 8 -> linear_v2_kernel<8>
    (300, 160, 4, 57, 32),   # vshrink 5: box 2, residual 2.5 -> linear_v_kernel<4, premul, 2>
    (61, 288, 4, 11, 32),    # vshrink 9: box 4 -> linear_v_kernel<4, premul, 4>
    (53, 544, 4, 10, 32),    # vshrink 17: box 8 -> linear_v_kernel<4, premul, 8>
    (53, 208, 4, 10, 32),    # vshrink 6.5: box 3 through the ring -> linear_v_kernel<4, premul, 0>
    (40, 608, 4, 8, 32),     # vshrink 19: box 9, loaded directly -> linear_v_kernel<4, premul, 0>
    (300, 128, 3, 57, 32),   # RGB, box 2 (residual 2.0, still the general kernel) -> linear_v_kernel<3, plain, 2>
    (61, 288, 3, 11, 32),    # RGB, box 4 -> linear_v_kernel<3, plain, 4>
    (53, 512, 3, 10, 32),    # RGB, box 8 -> linear_v_kernel<3, plain, 8>
    (53, 208, 3, 10, 32),    # RGB, box 3 -> linear_v_kernel<3, plain, 0>
    (40, 608, 3, 8, 32),     # RGB, box 9 -> linear_v_kernel<3, plain, 0>
]


def test_linear_sweep_reaches_every_v_form(oracle):
    """CPU: SWEEP launches every kernel V a plain linear plan can launch, and its RGBA frames put reduced alpha on both sides
    of unpremultiply's threshold: nonzero alpha with the colour zeroed, and alpha as low with the colour kept."""
    reachable = {("v", 4, 0, True), ("v", 4, 0, False), ("v", 4, 2, True), ("v", 4, 4, True), ("v", 4, 8, True),
                 ("v", 3, 0, False), ("v", 3, 2, False), ("v", 3, 4, False), ("v", 3, 8, False),
                 ("v2", 4, 2, True), ("v2", 4, 4, True), ("v2", 4, 8, True)}
    assert {v_form(*case) for case in SWEEP} == reachable
    for w, h, bands, tw, th in SWEEP:
        if bands == 4:
            t = oracle.thumbnail_image(sweep_frame(h, w, bands, 0), tw, th, size="force", linear=True)
            faint = (t[..., 3] > 0) & (t[..., 3] <= 3)
            dark = (t[..., :3] == 0).all(axis=-1)
            assert (faint & dark).any() and (faint & ~dark).any(), (w, h)


def test_oracle_rgba_correct_known_answer(oracle):
    t = oracle.thumbnail_image(FIX["rgba"], 64, linear=True)
    assert t.shape[:2] == tuple(FIX["correct_shape"][:2])
    assert abs(flatten_avg(t) - float(FIX["correct_avg"])) < 1


@pytest.mark.gpu
def test_gpu_rgba_correct_known_answer(vb, oracle):
    t = vb.Image(FIX["rgba"]).thumbnail_image(64, linear=True).numpy()
    assert abs(flatten_avg(t) - float(FIX["correct_avg"])) < 1
    assert np.array_equal(t, oracle.thumbnail_image(FIX["rgba"], 64, linear=True))


@pytest.mark.gpu
@pytest.mark.parametrize("shape,target,bands", [((512, 512), 64, 4), ((301, 517), 50, 4), ((400, 300), 60, 3),
                                                 ((640, 480), 111, 4)])
def test_gpu_linear_thumbnail_parity(vb, oracle, shape, target, bands):
    rng = np.random.default_rng(5)
    a = rng.integers(0, 256, shape + (bands,), dtype=np.uint8)
    got = vb.Image(a).thumbnail_image(target, linear=True).numpy()
    want = oracle.thumbnail_image(a, target, linear=True)
    assert got.shape == want.shape and np.array_equal(got, want)


def test_oracle_linear_chain_against_reference_sources():
    """CPU: the oracle's linear-light thumbnail against the reference's OWN sources under oracle/_ref --
    premultiply.c, resize.c (shrinkv / reducev / shrinkh / reduceh float branches), unpremultiply.c and the
    sRGB2scRGB / scRGB2sRGB line functions; only the 4th band's trip through vips_colour_build (x 1 / 255,
    x 255, cast) is restated here (colour.c:252-291)."""
    from oracle import pyoracle as orc
    from oracle import pyref
    if not pyref.available():
        pytest.skip("oracle/_ref not built")

    @pyref.recorded
    def reference_linear_thumbnail(a, target, height=None, size="both"):
        h, w, b = a.shape
        hs, vs, _, _ = orc.thumbnail_size(w, h, target, height, size)
        lin = pyref.colour_line("sRGB2scRGB", a[:, :, :3]).reshape(h, w, 3)
        if b == 4:
            alpha = (np.float32(1.0 / 255.0) * a[:, :, 3].astype(np.float32) + np.float32(0)).astype(np.float32)
            lin = np.concatenate([lin, alpha[:, :, None]], axis=2)
        im = pyref.RefImage.from_array(np.ascontiguousarray(lin), 28)
        if b == 4:
            im = im.premultiply()
        im = im.resize(1.0 / hs, 1.0 / vs)
        if b == 4:
            im = im.unpremultiply()
        res = im.numpy()
        rgb = pyref.colour_line("scRGB2sRGB", np.ascontiguousarray(res[:, :, :3])).reshape(res.shape[0], res.shape[1], 3)
        if b == 4:
            al = np.clip((np.float32(255.0) * res[:, :, 3] + np.float32(0)).astype(np.float32).astype(np.float64), 0, 255).astype(np.uint8)
            rgb = np.concatenate([rgb, al[:, :, None]], axis=2)
        return rgb

    rng = np.random.default_rng(77)
    for shape, target in (((256, 320, 4), 40), ((200, 150, 3), 33), ((333, 222, 4), 60)):
        a = rng.integers(0, 256, shape, dtype=np.uint8)
        assert np.array_equal(orc.thumbnail_image(a, target, linear=True), reference_linear_thumbnail(a, target)), shape
    # the geometry classes of the kernel sweep at a reduced size, on its frames (RGBA ones with the alpha-threshold block):
    # exact vertical shrinks 4, 8 and 16, a box of 9 rows, and RGB
    for w, h, bands, tw, th in ((40, 64, 4, 8, 16), (40, 128, 4, 8, 16), (40, 256, 4, 8, 16), (40, 304, 4, 8, 16),
                                (40, 128, 3, 8, 16), (40, 304, 3, 8, 16)):
        a = sweep_frame(h, w, bands, 0)
        want = reference_linear_thumbnail(a, tw, th, "force")
        assert np.array_equal(orc.thumbnail_image(a, tw, th, size="force", linear=True), want), (w, h, bands)


@pytest.mark.gpu
@pytest.mark.parametrize("shape,target,bands", [((2048, 2048), 256, 4), ((1024, 768), 128, 4), ((1200, 900), 150, 4),
                                                 ((1003, 2057), 120, 4), ((777, 555), 99, 3), ((4096, 512), 64, 4)])
def test_gpu_linear_two_kernel_path(vb, oracle, shape, target, bands):
    """the geometries of the uchar V4 cases through the linear-light kernels, and that they ARE the kernels"""
    rng = np.random.default_rng(6)
    a = rng.integers(0, 256, shape + (bands,), dtype=np.uint8)
    a[: shape[0] // 3, :, -1] = 0  # transparent band: unpremultiply's |alpha| < 0.01 branch
    plan = vb.ThumbnailPlan(shape[1], shape[0], bands, target, linear=True)
    assert plan.fused and plan.kernel == "linear_v_kernel + linear_h_kernel"
    n0 = vb.launch_count()
    got = plan.run_host(a[None])[0]
    assert vb.launch_count() - n0 == 2
    want = oracle.thumbnail_image(a, target, linear=True)
    assert got.shape == want.shape and np.array_equal(got, want)


@pytest.mark.gpu
def test_gpu_linear_batch_and_sharpen_stage(vb, oracle):
    from oracle import pyconv
    rng = np.random.default_rng(8)
    frames = rng.integers(0, 256, (5, 600, 800, 4), dtype=np.uint8)
    plan = vb.ThumbnailPlan(800, 600, 4, 100, linear=True)
    got = plan.run_host(frames)
    for i in range(5):
        assert np.array_equal(got[i], oracle.thumbnail_image(frames[i], 100, linear=True)), i
    plan.set_sharpen()
    got = plan.run_host(frames[:2])
    for i in range(2):
        assert np.array_equal(got[i], pyconv.sharpen(oracle.thumbnail_image(frames[i], 100, linear=True), "srgb")), i


@pytest.mark.gpu
@pytest.mark.parametrize("static", [True, False], ids=["static", "no_static"])
@pytest.mark.parametrize("w,h,bands,tw,th", SWEEP)
def test_gpu_linear_v_forms(vb, oracle, monkeypatch, w, h, bands, tw, th, static):
    """every kernel V form, bit for bit: one frame (rows split over CTAs, so CTAs start mid-frame) and a batch large enough
    that each CTA runs a whole frame; VB200_NO_LINEAR_STATIC puts the residual-2.0 geometries on the general kernel"""
    import torch
    if not static:
        monkeypatch.setenv("VB200_NO_LINEAR_STATIC", "1")
    plan = vb.ThumbnailPlan(w, h, bands, tw, th, size="force", linear=True)
    assert plan.fused and plan.kernel == "linear_v_kernel + linear_h_kernel"
    frames = [sweep_frame(h, w, bands, seed) for seed in (0, 1)]
    want = [oracle.thumbnail_image(f, tw, th, size="force", linear=True) for f in frames]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = -(-4 * sms // -(-w // 256))
    assert v_splits(w, plan.out_height, 1, sms) > 1 and v_splits(w, plan.out_height, n, sms) == 1
    for batch in (frames[:1], [frames[i % 2] for i in range(n)]):
        n0 = vb.launch_count()
        got = plan.run_host(np.stack(batch))
        assert vb.launch_count() - n0 == 2
        for i, g in enumerate(got):
            assert np.array_equal(g, want[i % 2]), (len(batch), i)


@pytest.mark.gpu
def test_gpu_linear_sub_batches(vb, oracle):
    """a batch whose float intermediate passes 2 GiB runs in sub-batches (16 frames of 128 MiB, then 2); frames alternate
    between two images and sit at a padded device stride.  A stride off the 4-byte grid is refused before any launch."""
    import torch
    w, h, tw, th = 4096, 2560, 512, 2048
    plan = vb.ThumbnailPlan(w, h, 4, tw, th, size="force", linear=True)
    assert plan.kernel == "linear_v_kernel + linear_h_kernel"
    n = 18
    assert n * plan.out_height * w * 4 * 4 > 2 << 30
    frames = [sweep_frame(h, w, 4, seed) for seed in (2, 3)]
    want = [oracle.thumbnail_image(f, tw, th, size="force", linear=True) for f in frames]
    fb, stride = plan.in_frame_bytes, plan.in_frame_bytes + 64
    src = [torch.from_numpy(f.reshape(-1)).cuda() for f in frames]
    din = torch.empty(n * stride, dtype=torch.uint8, device="cuda")
    for i in range(n):
        din[i * stride:i * stride + fb] = src[i % 2]
    dout = torch.full((n, plan.out_height, plan.out_width, 4), 77, dtype=torch.uint8, device="cuda")
    with pytest.raises(vb.Error, match="RGBA frames must be 4-byte aligned"):
        plan.run_device(din.data_ptr(), dout.data_ptr(), n, in_stride=fb + 2)
    torch.cuda.synchronize()
    assert bool((dout == 77).all())
    n0 = vb.launch_count()
    plan.run_device(din.data_ptr(), dout.data_ptr(), n, in_stride=stride)
    torch.cuda.synchronize()
    assert vb.launch_count() - n0 == 4
    got = dout.cpu().numpy()
    for i in range(n):
        assert np.array_equal(got[i], want[i % 2]), i


def h_shared_bytes(w, h, bands, tw, th):
    """kernel H's dynamic shared memory, the formula of linear_thumb_new (libvips_b200/csrc/thumbnail_linear.cu:661-662).
    Wse replays build_axis_table's positions in one rect; the plan restarts them per tile, which moves no position when
    the residual is exactly 2.0, as in the frames here."""
    from oracle import pyoracle as orc
    hs, _, ow, _ = orc.thumbnail_size(w, h, tw, th, "force")
    g = orc.reduce_geometry(w, 1.0 / max(1.0 / hs, 1.0 / w), "lanczos3", 2.0)
    assert g.residual == 2.0
    pos, first = 0.5 * g.residual - 0.5 - g.offset, []
    for _ in range(ow):
        first.append(int(pos))
        pos += g.residual
    wse = max(first) + g.n_point
    return 65 * g.n_point * 8 + 260 * 4 + ((wse * bands + 3) & ~3) * 4 + ((ow * bands + 3) & ~3) * 4


@pytest.mark.gpu
@pytest.mark.parametrize("ow,kernel", [(4100, "linear_v_kernel + linear_h_kernel"), (4101, "leaf kernels")])
def test_gpu_linear_h_shared_memory_edge(vb, oracle, ow, kernel):
    """short, wide frames whose kernel H needs just under 200 KB of shared memory (two kernels) and just over it (the leaf
    chain): both give the oracle's pixels"""
    w, h, th = 4 * ow, 8, 2
    smem = h_shared_bytes(w, h, 4, ow, th)
    assert (smem <= 200 * 1024) == (kernel != "leaf kernels") and abs(smem - 200 * 1024) <= 64
    a = sweep_frame(h, w, 4, 4)
    plan = vb.ThumbnailPlan(w, h, 4, ow, th, size="force", linear=True)
    assert plan.kernel == kernel
    got = plan.run_host(a[None])[0]
    assert np.array_equal(got, oracle.thumbnail_image(a, ow, th, size="force", linear=True))

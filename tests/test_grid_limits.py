"""Images taller than 65 535 rows and batches of more than 65 535 frames through every device entry point.

CUDA refuses a launch whose gridDim.y or gridDim.z exceeds 65 535.  The whole-image kernels take one CTA row per
image row (or per group of rows) and cap gridDim.y there, walking the rest of the rows in a loop; the batch paths
launch at most 32 768 frames at a time.  These cases cross each threshold with the cheapest shape that reaches it
(narrow images, tiny frames repeated) and compare with the plain reference the rest of the suite trusts for that op:
oracle.pyoracle (resample, premultiply, thumbnail, colourspace), oracle.pyconv (conv, sharpen, morph, rank, flatten),
the host ICC evaluator and libjpeg-turbo.  Also the other ends: a very wide image of 1 to 3 rows, and 1 x 1, 1 x 2
and 2 x 1 images with masks and windows as large as the image."""
import numpy as np
import pytest

from oracle import pyconv
from oracle import pyoracle as orc

pytestmark = pytest.mark.gpu

TALL = (65535, 65536, 70001)  # the last full grid, the first row past it, and a ragged remainder
SMALL = ((1, 1), (1, 2), (2, 1))  # (height, width)
G15 = pyconv.gaussmat(2.5, 0.2, True, "float")
MASK3 = np.array([[1.0, 2.0, 1.0], [2.0, 4.0, 2.0], [1.0, 2.0, 1.0]])
ROW7 = np.array([[1.0, -2.0, 3.0, 8.0, 3.0, -2.0, 1.0]])


def rnd(dt, shape, seed):
    rng = np.random.default_rng(seed)
    if np.dtype(dt).kind == "f":
        return (rng.random(shape) * 255).astype(dt)
    info = np.iinfo(dt)
    return rng.integers(info.min, int(info.max) + 1, shape, dtype=dt)


def same(got, want, what=""):
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    bad = got != want
    if got.dtype.kind == "f":
        bad &= ~(np.isnan(got) & np.isnan(want))
    assert not bad.any(), (what, np.argwhere(bad)[:5])


# ----------------------------------------------------------------------------------------------- resample


@pytest.mark.parametrize("h", TALL)
@pytest.mark.parametrize("dt,bands", [(np.uint8, 4), (np.uint8, 3), (np.uint16, 1), (np.int16, 2), (np.int32, 1), (np.float32, 3)])
def test_tall_resample(vb, h, dt, bands):
    a = rnd(dt, (h, 3, bands), h + bands)
    im = vb.Image(a)
    same(im.shrinkv(3).numpy(), orc.shrinkv(a, 3), "shrinkv")
    same(im.shrinkh(2).numpy(), orc.shrinkh(a, 2), "shrinkh")
    for f in (1.7, 2.0):
        same(im.reducev(f).numpy(), orc.reducev(a, f), ("reducev", f))
        same(im.reduceh(f).numpy(), orc.reduceh(a, f), ("reduceh", f))
    for sc in (0.6, 0.5):
        same(im.resize(sc).numpy(), orc.resize(a, sc), ("resize", sc))


@pytest.mark.parametrize("h", TALL)
def test_tall_reduce_uchar_rgba_kernels(vb, h):
    """the word-wise uchar kernels at these heights: reduceh's staged dp2a kernel takes one CTA row per image row (the
    vertical kernels run over output rows: the cases below make those taller than the grid)"""
    for w in (1, 4, 8):
        a = rnd(np.uint8, (h, w, 4), w)
        same(vb.Image(a).reducev(1.3).numpy(), orc.reducev(a, 1.3), ("reducev", w))
        same(vb.Image(a).reduceh(1.3).numpy(), orc.reduceh(a, 1.3), ("reduceh", w))
        same(vb.Image(a).shrinkv(2).numpy(), orc.shrinkv(a, 2), ("shrinkv", w))


@pytest.mark.parametrize("dt,bands", [(np.uint8, 4), (np.uint8, 3), (np.uint16, 1), (np.float32, 1)])
def test_shrinkv_output_taller_than_the_grid(vb, dt, bands):
    """shrinkv runs over output rows: more than 2 x 65 535 input rows (uchar x 4 elements takes the word-wise kernel)"""
    a = rnd(dt, (131075, 1, bands), 200 + bands)
    got = vb.Image(a).shrinkv(2).numpy()
    assert got.shape[0] > 65535
    same(got, orc.shrinkv(a, 2))


@pytest.mark.parametrize("dt,bands", [(np.uint8, 3), (np.uint16, 1), (np.int16, 2), (np.int32, 1), (np.float32, 1)])
def test_reducev_output_taller_than_the_grid(vb, dt, bands):
    """reducev runs over output rows: a factor close to 1 on 70 001 rows gives more than 65 535"""
    a = rnd(dt, (70001, 1, bands), 210 + bands)
    got = vb.Image(a).reducev(1.05).numpy()
    assert got.shape[0] > 65535
    same(got, orc.reducev(a, 1.05))


def test_conv_line_kernel_taller_than_the_grid(vb, monkeypatch):
    """the one-output-per-thread 1-D kernels (taken when the register-blocked ones are switched off)"""
    monkeypatch.setenv("VB200_NO_CONV_BLOCK", "1")
    a = rnd(np.float32, (70001, 2, 2), 220)
    for m, sc in ((ROW7, 12.0), (ROW7.T.copy(), 12.0)):
        same(vb.Image(a).conv(m, sc, 0, "float").numpy(), pyconv.conv(a, m, sc, 0, "float"), m.shape)


@pytest.mark.parametrize("w", [1, 4])
def test_reducev_past_the_grouped_row_limit(vb, w):
    """reducev's dp2a kernels take 4 output rows per CTA: an output taller than 4 x 65 535 = 262 140 rows"""
    a = rnd(np.uint8, (300000, w, 4), 300 + w)
    got = vb.Image(a).reducev(1.1).numpy()
    assert got.shape[0] > 262140
    same(got, orc.reducev(a, 1.1))


@pytest.mark.parametrize("h", TALL)
@pytest.mark.parametrize("dt", [np.uint8, np.uint16, np.float32])
def test_tall_premultiply(vb, h, dt):
    a = rnd(dt, (h, 2, 4), h)
    a[::7, :, 3] = 0
    modes = (False, True) if dt == np.uint8 else (False,)
    for uchar in modes:
        pre = vb.Image(a).premultiply(255.0, uchar=uchar).numpy()
        same(pre, orc.premultiply(a, 255.0, uchar=uchar), ("premultiply", uchar))
        same(vb.Image(pre).unpremultiply(255.0, uchar=uchar).numpy(), orc.unpremultiply(pre, 255.0, uchar=uchar), ("unpremultiply", uchar))


@pytest.mark.parametrize("h", [33000, 65536])
@pytest.mark.parametrize("dt,bands,kernel", [(np.uint8, 4, "lanczos3"), (np.uint8, 3, "lanczos3"), (np.float32, 1, "linear"),
                                             (np.uint16, 2, "nearest")])
def test_tall_upsize(vb, h, dt, bands, kernel):
    """resize up, affine kernels: the output is taller than 65 535 rows"""
    a = rnd(dt, (h, 2, bands), h + bands)
    got = vb.Image(a).resize(2.5, kernel=kernel).numpy()
    assert got.shape[0] > 65535
    same(got, orc.resize(a, 2.5, kernel=kernel))


def test_tall_upsize_per_pixel_bicubic_and_zoom(vb, monkeypatch):
    a = rnd(np.uint8, (40000, 3, 4), 41)
    same(vb.Image(a).resize(2.0, kernel="nearest").numpy(), orc.resize(a, 2.0, kernel="nearest"), "zoom")
    monkeypatch.setenv("VB200_NO_AFFINE_SEP", "1")  # the one-pixel-per-thread bicubic kernel instead of the separable one
    same(vb.Image(a).resize(1.8).numpy(), orc.resize(a, 1.8), "affine_bicubic_u8x4_kernel")


def test_upsize_past_the_separable_tile_limit(vb):
    """the separable bicubic kernel takes 32 output rows per CTA: an output taller than 32 x 65 535 rows"""
    a = rnd(np.uint8, (1100000, 1, 4), 42)
    got = vb.Image(a).resize(2.0).numpy()
    assert got.shape[0] > 32 * 65535
    same(got, orc.resize(a, 2.0))


# ---------------------------------------------------------------------------------------------------- conv



@pytest.mark.parametrize("h", TALL)
@pytest.mark.parametrize("dt", [np.uint8, np.int16, np.float32])
def test_tall_conv(vb, h, dt):
    a = rnd(dt, (h, 3, 2), h)
    for m, sc in ((MASK3, 16.0), (ROW7, 12.0), (ROW7.T.copy(), 12.0), (G15[0].T.copy(), G15[1])):
        for pr in ("float", "integer"):
            same(vb.Image(a).conv(m, sc, 0, pr).numpy(), pyconv.conv(a, m, sc, 0, pr), (m.shape, pr))
    m, sc, off = pyconv.gaussmat(2.0, 0.2, True, "float")
    same(vb.Image(a).convsep(m, sc, off, "float").numpy(), pyconv.convsep(a, m, sc, off, "float"), "convsep")
    for pr in ("float", "integer"):
        same(vb.Image(a).gaussblur(1.5, 0.2, pr).numpy(), pyconv.gaussblur(a, 1.5, 0.2, pr), ("gaussblur", pr))


@pytest.mark.parametrize("h", TALL)
def test_tall_conv_vector_mode(vb, h):
    a = rnd(np.uint8, (h, 4, 4), h)
    gi = pyconv.gaussmat(1.2, 0.2, False, "integer")
    try:
        vb.set_vector_convi(True)
        for m, sc in ((MASK3, 16.0), (gi[0], gi[1])):
            same(vb.Image(a).conv(m, sc, 0, "integer").numpy(), pyconv.conv(a, m, sc, 0, "integer", vector=True), m.shape)
    finally:
        vb.set_vector_convi(False)


def test_conv_column_masks_past_the_grouped_row_limit(vb):
    """the vertical register-blocked conv kernels take 8 rows per CTA: more than 8 x 65 535 = 524 280 rows, with a dense
    Gaussian column and a sparse one"""
    a = rnd(np.uint8, (530000, 1, 1), 7)
    sparse = np.array([[1.0], [0.0], [0.0], [3.0], [0.0], [2.0], [0.0]])
    for m, sc in ((G15[0].T.copy(), G15[1]), (sparse, 6.0)):
        same(vb.Image(a).conv(m, sc, 0, "float").numpy(), pyconv.conv(a, m, sc, 0, "float"), m.shape)


@pytest.mark.parametrize("h", TALL)
def test_tall_sharpen(vb, h):
    a = rnd(np.uint8, (h, 2, 3), h)
    same(vb.Image(a, "srgb").sharpen().numpy(), pyconv.sharpen(a, "srgb"), "srgb")
    labs = orc.colourspace(a, "labs", "srgb")
    same(vb.Image(labs, "labs").sharpen().numpy(), pyconv.sharpen(labs, "labs"), "labs")


# ------------------------------------------------------------------------------------ morphology, rank, flatten

CROSS = np.array([[128.0, 255.0, 128.0], [255.0, 255.0, 255.0], [128.0, 255.0, 128.0]])


@pytest.mark.parametrize("h", TALL)
def test_tall_morph_rank_flatten(vb, h):
    a = rnd(np.uint8, (h, 3, 2), h)
    a[a < 128] = 0
    for op in ("erode", "dilate"):
        same(vb.Image(a).morph(CROSS, op).numpy(), pyconv.morph(a, CROSS, op), op)
    same(vb.Image(a).median(3).numpy(), pyconv.median(a, 3), "median")
    same(vb.Image(a).rank(3, 5, 0).numpy(), pyconv.rank(a, 3, 5, 0), "rank")
    f = rnd(np.float32, (h, 2, 4), h + 1)
    same(vb.Image(f).rank(1, 3, 2).numpy(), pyconv.rank(f, 1, 3, 2), "rank float")
    rgba = rnd(np.uint8, (h, 2, 4), h + 2)
    same(vb.Image(rgba).flatten((10, 20, 30)).numpy(), pyconv.flatten(rgba, (10, 20, 30)), "flatten")


def test_rank_past_the_tile_row_limit(vb):
    """rank's tiles are 8 rows: more than 8 x 65 535 = 524 280 rows"""
    a = rnd(np.uint8, (530000, 3, 1), 8)
    same(vb.Image(a).median(3).numpy(), pyconv.median(a, 3))


def test_rank_one_row_tiles(vb):
    """a 1 x 400 window of 4-band floats does not fit a tile of 8 rows in shared memory: the tile drops to 1 row, one
    CTA row per image row"""
    a = rnd(np.float32, (66000, 1, 4), 9)
    same(vb.Image(a).rank(1, 400, 0).numpy(), pyconv.rank(a, 1, 400, 0), "min")
    same(vb.Image(a).rank(1, 400, 200).numpy(), pyconv.rank(a, 1, 400, 200), "median")


# --------------------------------------------------------------------------------------------- colour, ICC

# (source, destination, input dtype): shift-cast, cast, the two x4 kernels, the route kernel, the B_W and HSV rows
ROUTES = [("srgb", "rgb16", np.uint8), ("lab", "lab", np.float32), ("srgb", "lab", np.uint8), ("lab", "srgb", np.float32),
          ("srgb", "xyz", np.uint8), ("labs", "srgb", np.int16), ("srgb", "b-w", np.uint8), ("srgb", "hsv", np.uint8)]


@pytest.mark.parametrize("h", TALL)
@pytest.mark.parametrize("w", [1, 4])
def test_tall_colourspace(vb, h, w):
    base = rnd(np.uint8, (h, w, 3), h + w)
    for src, dst, dt in ROUTES:
        a = base if src == "srgb" else orc.colourspace(base, src, "srgb")
        assert a.dtype == dt
        same(vb.Image(a, src).colourspace(dst).numpy(), orc.colourspace(a, dst, src), (src, dst))


@pytest.mark.parametrize("h", [65536, 70001])
def test_tall_icc(vb, h):
    import icc_fixtures as F
    from test_icc import host_eval
    a = rnd(np.uint8, (h, 1, 3), h)
    rgb, ink = F.rgb_profile(), F.ink_profile()
    lab = vb.Image(a, "srgb").icc_import(rgb)
    assert np.abs(lab.array.reshape(-1, 3) - host_eval(0, a.reshape(-1, 3), rgb)).max() < 2e-3
    back = lab.icc_export(rgb).numpy()
    want = host_eval(1, lab.array.reshape(-1, 3), rgb).reshape(a.shape)
    assert np.abs(back.astype(int) - want.astype(int)).max() <= 1 and (back != want).mean() < 1e-3
    inks = vb.Image(a, "srgb").icc_transform(ink, rgb).numpy()
    want = host_eval(2, a.reshape(-1, 3), rgb, ink).reshape(h, 1, 4)
    assert np.abs(inks.astype(int) - want.astype(int)).max() <= 1


# ---------------------------------------------------------------------------------------------- thumbnails


def test_tall_thumbnail_unfused(vb):
    a = rnd(np.uint8, (70000, 64, 4), 10)
    assert not vb.ThumbnailPlan(64, 70000, 4, 128).fused  # VS > 256: the chain of leaf kernels
    same(vb.Image(a).thumbnail_image(128).numpy(), orc.thumbnail_image(a, 128))


def test_tall_thumbnail_fused(vb):
    a = rnd(np.uint8, (70000, 16, 4), 11)
    plan = vb.ThumbnailPlan(16, 70000, 4, 6, 1000, size="force")
    assert plan.fused
    same(plan.run_host(a[None])[0], orc.thumbnail_image(a, 6, 1000, size="force"))


def test_thumbnail_output_taller_than_the_grid(vb):
    a = rnd(np.uint8, (140003, 4, 4), 12)
    got = vb.Image(a).thumbnail_image(3, 66001, size="force").numpy()
    assert got.shape[0] == 66001
    same(got, orc.thumbnail_image(a, 3, 66001, size="force"))


def test_tall_thumbnail_linear(vb):
    a = rnd(np.uint8, (70001, 8, 4), 13)
    same(vb.Image(a).thumbnail_image(5, 30000, size="force", linear=True).numpy(),
         orc.thumbnail_image(a, 5, 30000, size="force", linear=True))


def test_tall_chain(vb):
    """a Chain pumps its steps through its own code: resize, integer Gaussian blur and dilation on 70 001 rows"""
    a = rnd(np.uint8, (70001, 3, 3), 14)
    got = vb.Chain().resize(0.9).gaussblur(1.2, 0.2, "integer").morph(CROSS, "dilate").run([a])[0].numpy()
    want = pyconv.morph(pyconv.gaussblur(orc.resize(a, 0.9), 1.2, 0.2, "integer"), CROSS, "dilate")
    same(got, want)


# ------------------------------------------------------------------------------------------ the other ends


def test_wide_few_rows(vb):
    for h in (1, 2, 3):
        a = rnd(np.uint8, (h, 70001, 4), h)
        im = vb.Image(a)
        same(im.shrinkh(3).numpy(), orc.shrinkh(a, 3), ("shrinkh", h))
        same(im.reduceh(1.7).numpy(), orc.reduceh(a, 1.7), ("reduceh", h))
        same(im.resize(0.6).numpy(), orc.resize(a, 0.6), ("resize", h))
        same(im.resize(1.5).numpy(), orc.resize(a, 1.5), ("upsize", h))
        same(im.premultiply(255.0).numpy(), orc.premultiply(a, 255.0), ("premultiply", h))
        same(im.conv(MASK3, 16.0, 0, "integer").numpy(), pyconv.conv(a, MASK3, 16.0, 0, "integer"), ("conv", h))
        same(im.gaussblur(1.5, 0.2, "float").numpy(), pyconv.gaussblur(a, 1.5, 0.2, "float"), ("gaussblur", h))
        same(im.morph(CROSS, "dilate").numpy(), pyconv.morph(a, CROSS, "dilate"), ("morph", h))
        same(im.rank(3, h, 0).numpy(), pyconv.rank(a, 3, h, 0), ("rank", h))
        same(im.flatten((1, 2, 3)).numpy(), pyconv.flatten(a, (1, 2, 3)), ("flatten", h))
        rgb = np.ascontiguousarray(a[..., :3])
        for src, dst, _ in ROUTES[2:]:
            x = rgb if src == "srgb" else orc.colourspace(rgb, src, "srgb")
            same(vb.Image(x, src).colourspace(dst).numpy(), orc.colourspace(x, dst, src), (src, dst, h))


@pytest.mark.parametrize("h,w", SMALL)
def test_smallest_images(vb, h, w):
    a = rnd(np.uint8, (h, w, 4), h * 3 + w)
    im = vb.Image(a)
    for m, sc in ((MASK3, 16.0), (G15[0], G15[1]), (G15[0].T.copy(), G15[1])):  # 15 taps over a 1- or 2-pixel image
        for pr in ("float", "integer"):
            same(im.conv(m, sc, 0, pr).numpy(), pyconv.conv(a, m, sc, 0, pr), (m.shape, pr))
    same(im.gaussblur(1.5, 0.2, "integer").numpy(), pyconv.gaussblur(a, 1.5, 0.2, "integer"), "gaussblur")
    same(im.morph(CROSS, "erode").numpy(), pyconv.morph(a, CROSS, "erode"), "morph")
    for idx in range(w * h):
        same(im.rank(w, h, idx).numpy(), pyconv.rank(a, w, h, idx), ("rank = image", idx))
    same(im.premultiply(255.0, uchar=True).numpy(), orc.premultiply(a, 255.0, uchar=True), "premultiply")
    same(im.flatten((9, 8, 7)).numpy(), pyconv.flatten(a, (9, 8, 7)), "flatten")
    same(im.resize(3.0).numpy(), orc.resize(a, 3.0), "upsize")
    same(im.resize(2.0, kernel="nearest").numpy(), orc.resize(a, 2.0, kernel="nearest"), "zoom")
    rgb = np.ascontiguousarray(a[..., :3])
    for src, dst, _ in ROUTES:
        x = rgb if src == "srgb" else orc.colourspace(rgb, src, "srgb")
        same(vb.Image(x, src).colourspace(dst).numpy(), orc.colourspace(x, dst, src), (src, dst))
    same(vb.Image(rgb, "srgb").sharpen().numpy(), pyconv.sharpen(rgb, "srgb"), "sharpen")


# ------------------------------------------------------------------------------------------------ frames

NF = 70001  # frames in one device call: more than 65 535


def run_frames(vb, plan, base):
    """NF frames, base[i % len(base)], through one run_device call on torch-held buffers"""
    import torch
    idx = np.arange(NF) % len(base)
    din = torch.from_numpy(base).cuda()[torch.from_numpy(idx).cuda()].contiguous()
    dout = torch.zeros((NF, plan.out_height, plan.out_width, plan.bands), dtype=torch.uint8, device="cuda")
    vb.set_stream(torch.cuda.current_stream().cuda_stream)
    try:
        plan.run_device(din.data_ptr(), dout.data_ptr(), NF)
        torch.cuda.synchronize()
    finally:
        vb.set_stream(0)
    return dout.cpu().numpy(), idx


@pytest.mark.parametrize("bands,linear", [(4, True), (3, False), (4, False)])
def test_many_frames_one_call(vb, bands, linear):
    base = rnd(np.uint8, (4, 32, 32, bands), bands + linear)
    plan = vb.ThumbnailPlan(32, 32, bands, 12, linear=linear)
    assert plan.fused
    if linear:
        assert plan.kernel == "linear_v_kernel + linear_h_kernel"
    got, idx = run_frames(vb, plan, base)
    want = np.stack([orc.thumbnail_image(f, 12, linear=linear) for f in base])
    same(got, want[idx])


def test_jpeg_decode_many_frames(vb):
    from test_jpeg import encode, synth, turbo_decode
    streams = [encode(synth(8, 16, seed=i), 85, 2) for i in range(4)]
    assert all(b"\xff\xdd" not in s for s in streams)  # no restart interval: one interval per frame
    got = vb.jpeg_decode_batch([streams[i % 4] for i in range(NF)])
    want = np.stack([turbo_decode(s, 1) for s in streams])
    same(got, want[np.arange(NF) % 4])


def test_jpegsave_many_frames(vb):
    from test_jpeg import synth
    from test_jpeg_encode import turbo_encode
    base = np.stack([synth(8, 8, seed=i) for i in range(4)])
    got = vb.jpegsave_batch(base[np.arange(NF) % 4], 75)
    want = [turbo_encode(f, 75, 2) for f in base]
    bad = [i for i in range(NF) if got[i] != want[i % 4]]
    assert not bad, bad[:5]

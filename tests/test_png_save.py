"""PNG save (csrc/png_encode.cu): vips_pngsave_buffer's 8-bit frames deflated on the device.

The CPU half pins the host twin -- the same per-position, per-symbol and per-block code the kernels run -- to Python's zlib
(window bits 15, memLevel 8) at levels 4-9 with both strategies, and its PNG framing to a chunk walk, Pillow and the project's
own decoder.  The GPU half pins the device streams to the host twin byte for byte."""
import ctypes as C
import io
import struct
import threading
import zlib

import numpy as np
import pytest
from PIL import Image as PIL

import libvips_b200 as vb

LEVELS = range(4, 10)
STRATEGIES = [("default", zlib.Z_DEFAULT_STRATEGY), ("filtered", zlib.Z_FILTERED)]


def zlib_stream(data, level, strategy):
    c = zlib.compressobj(level, zlib.DEFLATED, 15, 8, strategy)
    return c.compress(data) + c.flush()


def zlib_rows(rows, level, strategy):
    """what libspng does: one compress call per scanline"""
    c = zlib.compressobj(level, zlib.DEFLATED, 15, 8, strategy)
    return b"".join(c.compress(r) for r in rows) + c.flush()


def corpus():
    rng = np.random.default_rng(7)
    yy, xx = np.mgrid[0:160, 0:200]
    smooth = (np.sin(xx / 13.0) + np.cos(yy / 19.0)) * 60 + 128
    out = {
        "noise": rng.integers(0, 256, 20000, dtype=np.uint8).tobytes(),
        "photo": np.clip(smooth + rng.normal(0, 5, smooth.shape), 0, 255).astype(np.uint8).tobytes(),
        "flat": bytes(40000),
        "quantised": (smooth // 16 * 16).astype(np.uint8).tobytes(),
        "periodic": (np.arange(60000) % 7 * 31 % 256).astype(np.uint8).tobytes(),
        "periodic-long": np.tile(rng.integers(0, 256, 300, dtype=np.uint8), 120).tobytes(),
        "runs-to-end": rng.integers(0, 256, 1000, dtype=np.uint8).tobytes() + b"\x05" * 700,
        "incompressible": rng.integers(0, 256, 70000, dtype=np.uint8).tobytes(),
        "lowentropy": rng.integers(0, 3, 90000, dtype=np.uint8).tobytes(),
        # 16383 literals and more: blocks cut where zlib's symbol buffer fills
        "literals-16383": rng.permutation(np.arange(16383 + 3) % 256).astype(np.uint8).tobytes(),
    }
    for n in list(range(0, 12)) + [37, 100, 255, 256, 257, 258, 259, 260, 261, 262, 263, 299, 300]:
        out["small-%d" % n] = rng.integers(0, 4, n, dtype=np.uint8).tobytes()
    # four-symbol noise over 64 KiB: at levels 8-9 the hash chains run out at the window limit (a later candidate exactly
    # MAX_DIST back ends zlib's walk) before they run out of max_chain
    for seed in (0, 9):
        r = np.random.default_rng(seed)
        n = int(r.integers(64 * 1024, 200 * 1024))
        out["maxdist-%d" % seed] = r.integers(0, 4, n).astype(np.uint8).tobytes()
    base = np.clip(smooth.ravel() + rng.normal(0, 2, smooth.size), 0, 255).astype(np.uint8)
    for n in (32768 - 1, 32768, 32768 + 300, 65274, 65280, 65536, 65536 + 250, 98304 + 7):
        tail = np.resize(base, n).tobytes()
        out["window-%d" % n] = tail
        out["window-run-%d" % n] = tail[:-300] + tail[-600:-300]
    return out


CORPUS = corpus()


@pytest.mark.parametrize("name", sorted(CORPUS))
def test_deflate_twin_equals_zlib(name):
    data = CORPUS[name]
    for level in LEVELS:
        for sname, st in STRATEGIES:
            want = zlib_stream(data, level, st)
            got = vb.deflate_host_twin(data, level, sname)
            assert got == want, "%s level %d %s: %d vs %d bytes" % (name, level, sname, len(got), len(want))


@pytest.mark.parametrize("name", ["photo", "quantised", "window-65536", "window-98311", "periodic-long"])
def test_zlib_row_fed_equals_one_shot(name):
    data = CORPUS[name]
    rows = [data[i:i + 777] for i in range(0, len(data), 777)]
    for level in LEVELS:
        for _, st in STRATEGIES:
            assert zlib_rows(rows, level, st) == zlib_stream(data, level, st)


def test_stored_blocks_are_chosen_for_incompressible_data():
    z = vb.deflate_host_twin(CORPUS["incompressible"], 6)
    assert len(z) > len(CORPUS["incompressible"])
    assert z[2] & 6 == 0  # the first block is stored


# ------------------------------------------------------------------------------------------------------------ framing

def chunks(png):
    assert png[:8] == b"\x89PNG\r\n\x1a\n"
    at, out = 8, []
    while at < len(png):
        n, = struct.unpack(">I", png[at:at + 4])
        kind, data = png[at + 4:at + 8], png[at + 8:at + 8 + n]
        crc, = struct.unpack(">I", png[at + 8 + n:at + 12 + n])
        assert crc == zlib.crc32(kind + data) & 0xFFFFFFFF, kind
        out.append((kind, data))
        at += 12 + n
    assert at == len(png)
    return out


def frame(h, w, bands, seed=0, kind="photo"):
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rng.integers(0, 256, (h, w, bands), dtype=np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    base = (np.sin(xx / 9.0 + seed) + np.cos(yy / 7.0)) * 50 + 120
    return np.clip(base[..., None] + rng.normal(0, 4, (h, w, bands)), 0, 255).astype(np.uint8)


def scanlines(a):
    return b"".join(b"\0" + row.tobytes() for row in a)


@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 1, 4), (7, 5, 2), (33, 17, 3), (64, 129, 4), (300, 301, 1), (150, 97, 3)])
def test_png_twin_framing(shape):
    h, w, b = shape
    a = frame(h, w, b, seed=h + w)
    for level in (4, 6, 9):
        for sname, st in STRATEGIES:
            png = vb.pngsave_host_twin(a, level, sname, xres=2.8346)
            cs = chunks(png)
            kinds = [k for k, _ in cs]
            assert kinds[0] == b"IHDR" and kinds[1] == b"pHYs" and kinds[-1] == b"IEND"
            assert set(kinds[2:-1]) == {b"IDAT"}
            ihdr = cs[0][1]
            assert struct.unpack(">IIBBBBB", ihdr) == (w, h, 8, [0, 0, 4, 2, 6][b], 0, 0, 0)
            assert cs[1][1] == struct.pack(">IIB", 2835, 2835, 1)
            idat = [d for k, d in cs if k == b"IDAT"]
            assert all(len(d) <= 8192 for d in idat) and all(len(d) == 8192 for d in idat[:-1])
            assert b"".join(idat) == zlib_stream(scanlines(a), level, st)
            assert np.array_equal(vb.png_decode_host_twin(png), a)
            assert np.array_equal(np.asarray(PIL.open(io.BytesIO(png))).reshape(h, w, b), a)


def test_png_twin_profile():
    a = frame(20, 30, 3)
    prof = bytes(range(256)) * 13
    png = vb.pngsave_host_twin(a, 6, profile=prof)
    cs = chunks(png)
    assert [k for k, _ in cs][:3] == [b"IHDR", b"iCCP", b"pHYs"]
    name, rest = cs[1][1].split(b"\0", 1)
    assert name == b"icc" and rest[0] == 0
    assert zlib.decompress(rest[1:]) == prof
    assert vb.png_icc_profile(png) == prof
    assert PIL.open(io.BytesIO(png)).info.get("icc_profile") == prof


def test_png_twin_multi_idat():
    a = frame(200, 200, 4, kind="noise")
    cs = chunks(vb.pngsave_host_twin(a))
    assert sum(k == b"IDAT" for k, _ in cs) > 10


@pytest.mark.parametrize("args,reason", [
    (dict(compression=3), "compression 3"), (dict(compression=0), "compression 0"), (dict(compression=10), "compression 10"),
    (dict(strategy=2), "strategy 2"), (dict(xres=float("nan")), "xres"),
])
def test_declined_options(args, reason):
    with pytest.raises(vb.Error, match=reason):
        vb.pngsave_host_twin(np.zeros((2, 2, 3), np.uint8), **args)
    with pytest.raises(vb.Error, match=reason):
        vb.deflate_host_twin(b"abc", args.get("compression", 6), args.get("strategy", "default")) if "xres" not in args else \
            vb.pngsave_host_twin(np.zeros((2, 2, 1), np.uint8), **args)


def test_declined_bands_and_size():
    with pytest.raises(vb.Error, match="5 bands"):
        vb.pngsave_host_twin(np.zeros((2, 2, 5), np.uint8))
    L = vb.lib()
    opts = vb.PngSaveOptions(6, 0, 1.0)
    n = C.c_size_t()
    assert L.vb200_debug_png_encode(b"\0" * 16, 1 << 20, 1 << 15, (1 << 13) + 1, 1, C.byref(opts), None, 0, None, 0, C.byref(n)) == -1
    assert b"2^28 pixels" in L.vb200_error_buffer()
    L.vb200_error_clear()


def test_declined_format():
    img = vb.Image(np.zeros((2, 2, 3), np.uint16))
    with pytest.raises(vb.Error, match="uchar"):
        img.pngsave_buffer()


def test_abi_names_resolve():
    L = vb.lib()
    for name in ("vb200_pngsave_batch", "vb200_pngsave_buffer", "vb200_debug_png_encode", "vb200_debug_deflate"):
        assert getattr(L, name) is not None


# ---------------------------------------------------------------------------------------------------------------- GPU

@pytest.fixture(scope="module")
def gpu():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    vb.init(0)
    return torch


@pytest.mark.gpu
def test_device_equals_twin_mixed(gpu):
    for b in (1, 2, 3, 4):
        for shape in ((1, 1), (17, 13), (64, 64), (131, 257)):
            frames = np.stack([frame(*shape, b, seed=s, kind="noise" if s == 2 else "photo") for s in range(4)])
            for level, sname in ((6, "default"), (4, "filtered"), (9, "default")):
                got = vb.pngsave_batch(frames, level, sname, xres=3.0)
                for i in range(len(frames)):
                    assert got[i] == vb.pngsave_host_twin(frames[i], level, sname, xres=3.0), (b, shape, level, sname, i)


@pytest.mark.gpu
def test_device_chains_to_the_window_limit(gpu):
    """four-symbol noise: chains at levels 8-9 reach MAX_DIST before max_chain; the device's IDATs are zlib's stream"""
    frames = np.random.default_rng(5).integers(0, 4, (3, 300, 400, 1)).astype(np.uint8)
    for level in (8, 9):
        for sname, st in STRATEGIES:
            for i, png in enumerate(vb.pngsave_batch(frames, level, sname)):
                idat = b"".join(d for k, d in chunks(png) if k == b"IDAT")
                assert idat == zlib_stream(scanlines(frames[i]), level, st), (level, sname, i)


@pytest.mark.gpu
def test_device_large_frames_cross_window_slides(gpu):
    frames = np.stack([frame(300, 250, 3, seed=s) for s in range(2)] + [np.zeros((300, 250, 3), np.uint8)])
    got = vb.pngsave_batch(frames, 6)
    for i in range(3):
        assert got[i] == vb.pngsave_host_twin(frames[i], 6)


@pytest.mark.gpu
def test_device_memory_strides_and_profile(gpu):
    torch = gpu
    a = np.stack([frame(23, 19, 3, seed=s) for s in range(5)])
    big = np.zeros((5, 23 + 3, 19 * 3 + 7), np.uint8)
    big[:, :23, 1:1 + 19 * 3] = a.reshape(5, 23, -1)
    t = torch.from_numpy(big).cuda()
    L = vb.lib()
    opts = vb.PngSaveOptions(6, 0, 1.0)
    prof = b"profile" * 50
    stride = 1 << 16
    out = np.zeros((5, stride), np.uint8)
    lens = (C.c_size_t * 5)()
    bpl, fs = big.shape[2], big.shape[1] * big.shape[2]
    rc = L.vb200_pngsave_batch(C.c_void_p(t.data_ptr() + 1), vb.DEVICE, bpl, fs, 5, 19, 23, 3, C.byref(opts), prof, len(prof),
                               out.ctypes.data_as(C.c_void_p), vb.HOST, stride, lens)
    assert rc == 0, L.vb200_error_buffer()
    for i in range(5):
        assert out[i, :lens[i]].tobytes() == vb.pngsave_host_twin(a[i], 6, profile=prof)
    # host frames at the same odd strides, device output
    dout = torch.zeros((5, stride), dtype=torch.uint8, device="cuda")
    rc = L.vb200_pngsave_batch(C.c_void_p(big.ctypes.data + 1), vb.HOST, bpl, fs, 5, 19, 23, 3, C.byref(opts), prof, len(prof),
                               C.c_void_p(dout.data_ptr()), vb.DEVICE, stride, lens)
    assert rc == 0, L.vb200_error_buffer()
    back = dout.cpu().numpy()
    for i in range(5):
        assert back[i, :lens[i]].tobytes() == vb.pngsave_host_twin(a[i], 6, profile=prof)


@pytest.mark.gpu
def test_device_grid_limits(gpu):
    many = np.random.default_rng(3).integers(0, 3, (70001, 1, 2, 1), dtype=np.uint8)
    got = vb.pngsave_batch(many, 6)
    for i in (0, 1, 32767, 32768, 65535, 70000):
        assert got[i] == vb.pngsave_host_twin(many[i], 6)
    tall = np.random.default_rng(4).integers(0, 2, (1, 70001, 1, 1), dtype=np.uint8)
    assert vb.pngsave_batch(tall, 6)[0] == vb.pngsave_host_twin(tall[0], 6)


@pytest.mark.gpu
def test_device_tiny_budget_chunks(gpu):
    frames = np.stack([frame(40, 40, 4, seed=s) for s in range(9)])
    L = vb.lib()
    try:
        L.vb200_debug_png_set_budget(1 << 20)
        got = vb.pngsave_batch(frames, 7)
    finally:
        L.vb200_debug_png_set_budget(0)
    for i in range(9):
        assert got[i] == vb.pngsave_host_twin(frames[i], 7)


@pytest.mark.gpu
def test_device_overflow_writes_nothing_and_pool(gpu):
    L = vb.lib()
    L.vb200_debug_dz_pool_used.restype = C.c_size_t
    frames = np.stack([np.zeros((30, 30, 3), np.uint8), frame(30, 30, 3, kind="noise")])
    vb.pngsave_batch(frames, 6)
    pool = L.vb200_debug_dz_pool_used()
    small = len(vb.pngsave_host_twin(frames[0], 6)) + 10
    out = np.full((2, small), 0xA5, np.uint8)
    lens = (C.c_size_t * 2)()
    opts = vb.PngSaveOptions(6, 0, 1.0)
    rc = L.vb200_pngsave_batch(frames.ctypes.data_as(C.c_void_p), vb.HOST, 90, 2700, 2, 30, 30, 3, C.byref(opts), None, 0,
                               out.ctypes.data_as(C.c_void_p), vb.HOST, small, lens)
    assert rc == -1 and b"frame 1" in L.vb200_error_buffer()
    L.vb200_error_clear()
    assert (out == 0xA5).all()
    assert L.vb200_debug_dz_pool_used() == pool
    vb.pngsave_batch(frames, 6)
    assert L.vb200_debug_dz_pool_used() == pool


@pytest.mark.gpu
def test_device_two_threads(gpu):
    a = np.stack([frame(50, 60, 4, seed=s) for s in range(6)])
    b = np.stack([frame(33, 71, 1, seed=s) for s in range(6)])
    res = {}

    def run(key, x):
        res[key] = vb.pngsave_batch(x, 6)

    ts = [threading.Thread(target=run, args=(k, x)) for k, x in (("a", a), ("b", b))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert [vb.pngsave_host_twin(x, 6) for x in a] == res["a"]
    assert [vb.pngsave_host_twin(x, 6) for x in b] == res["b"]


@pytest.mark.gpu
def test_png_thumbnail_resave(gpu):
    torch = gpu
    from oracle import pyoracle
    srcs = [frame(200, 160, 4, seed=s) for s in range(3)]
    streams = []
    for s in srcs:
        buf = io.BytesIO()
        PIL.fromarray(s).save(buf, "PNG")
        streams.append(buf.getvalue())
    plan = vb.ThumbnailPlan(160, 200, 4, 64)
    th = plan.run_png(streams)
    want = [pyoracle.thumbnail_image(s, 64) for s in srcs]
    for i in range(3):
        assert np.array_equal(th[i], want[i])
    got = vb.pngsave_batch(np.stack(th), 6)
    assert got == [vb.pngsave_host_twin(w, 6) for w in want]


@pytest.mark.gpu
def test_device_round_trip(gpu):
    a = np.stack([frame(45, 77, 2, seed=s) for s in range(4)])
    got = vb.pngsave_batch(a, 5, "filtered")
    assert np.array_equal(vb.png_decode_batch(got), a)
    img = vb.Image(a[0])
    assert img.pngsave_buffer(5, "filtered") == got[0]

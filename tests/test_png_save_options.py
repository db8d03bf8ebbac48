"""PNG save's scanline options (csrc/png_encode.cu): vips_pngsave's filter, interlace and bitdepth.

The CPU half builds the scanlines here from the PNG specification (2nd edition: 9.2's filters on raw bytes, 8.2's Adam7
passes) and from spngsave.c's rules (vips_foreign_save_spng_pack, its tail included), deflates them with Python's zlib, and
pins the host twin's IDAT payloads to that stream; Pillow decodes every stream.  The GPU half pins the device streams to
the host twin byte for byte."""
import ctypes as C
import io
import struct
import zlib

import numpy as np
import pytest
from PIL import Image as PIL

import libvips_b200 as vb

FILTERS = {"none": 0, "sub": 1, "up": 2, "avg": 3, "paeth": 4}
ADAM7 = [(0, 0, 8, 8), (4, 0, 8, 8), (0, 4, 4, 8), (2, 0, 4, 4), (0, 2, 2, 4), (1, 0, 2, 2), (0, 1, 1, 2)]
SETTINGS = [(6, "default", zlib.Z_DEFAULT_STRATEGY), (4, "filtered", zlib.Z_FILTERED), (9, "default", zlib.Z_DEFAULT_STRATEGY),
            (6, "filtered", zlib.Z_FILTERED), (4, "default", zlib.Z_DEFAULT_STRATEGY), (9, "filtered", zlib.Z_FILTERED)]
SIZES = [(h, w) for h in range(1, 10) for w in range(1, 10)] + [(17, 33), (64, 64)]


# ------------------------------------------------------------------------------------------------ the model, restated

def passes(a, interlace):
    """the non-empty passes of a [h, w, bands] frame: Adam7's sub-images, or the frame"""
    for x0, y0, dx, dy in (ADAM7 if interlace else [(0, 0, 1, 1)]):
        sub = a[y0::dy, x0::dx]
        if sub.shape[0] and sub.shape[1]:
            yield sub


def pack(row, depth):
    """vips_foreign_save_spng_pack (spngsave.c:295-324) of one row of grey samples, line by line"""
    pixel_mask = 8 // depth - 1
    bits, out = 0, []
    for x, p in enumerate(row):
        bits = ((bits << depth) | (int(p) >> (8 - depth))) & 0xFF
        if (x & pixel_mask) == pixel_mask:
            out.append(bits)
    x = len(row)
    if x & pixel_mask:
        collected_bits = (x & pixel_mask) << (depth - 1)
        out.append((bits << (8 - collected_bits)) & 0xFF)
    return bytes(out)


def filter_row(raw, prev, ft, bpp):
    """PNG 2nd edition 9.2: a = left by bpp, b = above, c = above-left, 0 where absent"""
    r = np.frombuffer(raw, np.uint8).astype(np.int32)
    b = np.frombuffer(prev, np.uint8).astype(np.int32) if prev is not None else np.zeros_like(r)
    a, c = np.zeros_like(r), np.zeros_like(r)
    a[bpp:], c[bpp:] = r[:-bpp], b[:-bpp]
    if ft == 0:
        pred = np.zeros_like(r)
    elif ft == 1:
        pred = a
    elif ft == 2:
        pred = b
    elif ft == 3:
        pred = (a + b) >> 1
    else:
        p = a + b - c
        pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
        pred = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
    return bytes([ft]) + ((r - pred) & 0xFF).astype(np.uint8).tobytes()


def scan_rows(a, filter="none", interlace=False, bitdepth=8):
    """every scanline of a frame, pass by pass and row by row"""
    a = a if a.ndim == 3 else a[..., None]
    ft, bpp = FILTERS[filter], (a.shape[2] if bitdepth == 8 else 1)
    rows = []
    for sub in passes(a, interlace):
        prev = None
        for y in range(sub.shape[0]):
            raw = sub[y].tobytes() if bitdepth == 8 else pack(sub[y, :, 0], bitdepth)
            rows.append(filter_row(raw, prev, ft, bpp))
            prev = raw
    return rows


def zlib_stream(data, level, strategy):
    c = zlib.compressobj(level, zlib.DEFLATED, 15, 8, strategy)
    return c.compress(data) + c.flush()


def chunks(png):
    assert png[:8] == b"\x89PNG\r\n\x1a\n"
    at, out = 8, []
    while at < len(png):
        n, = struct.unpack(">I", png[at:at + 4])
        kind, data = png[at + 4:at + 8], png[at + 8:at + 8 + n]
        assert struct.unpack(">I", png[at + 8 + n:at + 12 + n])[0] == zlib.crc32(kind + data) & 0xFFFFFFFF, kind
        out.append((kind, data))
        at += 12 + n
    assert at == len(png)
    return out


def idat(png):
    return b"".join(d for k, d in chunks(png) if k == b"IDAT")


def frame(h, w, bands, seed=0, kind="noise"):
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rng.integers(0, 256, (h, w, bands), dtype=np.uint8)
    if kind == "flat":
        return np.full((h, w, bands), rng.integers(0, 256), np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    base = (np.sin(xx / 9.0 + seed) + np.cos(yy / 7.0)) * 50 + 120
    return np.clip(base[..., None] + rng.normal(0, 4, (h, w, bands)), 0, 255).astype(np.uint8)


def low_bit_expected(a, depth):
    """what a reader gets back from spngsave's packed grey: samples scaled to 8 bits; at depth 4 an odd-width row's last
    pixel is its left neighbour's (0 for a one-pixel row), since the pack's tail shifts by 0 there"""
    v = (a[..., 0].astype(np.int32) >> (8 - depth)) * (255 // ((1 << depth) - 1))
    w = a.shape[1]
    if depth == 4 and w % 2:
        v[:, w - 1] = v[:, w - 2] if w > 1 else 0
    return v.astype(np.uint8)


# ---------------------------------------------------------------------------------------------------------------- CPU

@pytest.mark.parametrize("bands", [1, 2, 3, 4])
@pytest.mark.parametrize("interlace", [False, True])
@pytest.mark.parametrize("filter", sorted(FILTERS))
def test_zlib_stream_every_filter_and_size(filter, interlace, bands):
    """every size from 1 x 1 to 9 x 9 covers every empty Adam7 pass; levels and strategies are sampled, not multiplied"""
    for i, (h, w) in enumerate(SIZES):
        for kind in ("noise", "flat"):
            a = frame(h, w, bands, seed=i, kind=kind)
            level, sname, st = SETTINGS[(i + len(kind) + FILTERS[filter] + bands) % len(SETTINGS)]
            png = vb.pngsave_host_twin(a, level, sname, filter=filter, interlace=interlace)
            want = zlib_stream(b"".join(scan_rows(a, filter, interlace)), level, st)
            assert idat(png) == want, (h, w, kind, level, sname)


@pytest.mark.parametrize("depth", [1, 2, 4])
def test_low_bitdepth_every_leftover(depth):
    for w in range(1, 18):
        for h in (1, 2, 5):
            for kind in ("noise", "flat", "photo"):
                a = frame(h, w, 1, seed=w * 7 + h, kind=kind)
                level, sname, st = SETTINGS[(w + h) % len(SETTINGS)]
                png = vb.pngsave_host_twin(a, level, sname, bitdepth=depth)
                assert idat(png) == zlib_stream(b"".join(scan_rows(a, bitdepth=depth)), level, st), (w, h, kind)
                got = np.asarray(PIL.open(io.BytesIO(png)).convert("L"))
                assert np.array_equal(got, low_bit_expected(a, depth)), (w, h, kind)


def test_depth4_tail_keeps_the_last_sample_in_the_padding():
    """spngsave's tail at depth 4 writes v[w-2] << 4 | v[w-1]: the last pixel reads as its left neighbour"""
    a = np.array([[[0x10], [0x20], [0xF0]]], np.uint8)
    rows = scan_rows(a, bitdepth=4)
    assert rows == [b"\x00\x12\x2F"]
    assert zlib.decompress(idat(vb.pngsave_host_twin(a, bitdepth=4))) == b"\x00\x12\x2F"
    one = np.array([[[0xA0]]], np.uint8)
    assert zlib.decompress(idat(vb.pngsave_host_twin(one, bitdepth=4))) == b"\x00\x0A"


@pytest.mark.parametrize("filter", sorted(FILTERS))
def test_zlib_row_fed_equals_one_shot(filter):
    """libspng feeds zlib one scanline at a time; on this corpus that stream is the one-shot stream"""
    for interlace in (False, True):
        for shape in ((64, 64, 3), (17, 33, 4), (150, 97, 1), (120, 200, 2)):
            rows = scan_rows(frame(*shape, seed=sum(shape), kind="photo"), filter, interlace)
            for level, _, st in SETTINGS:
                c = zlib.compressobj(level, zlib.DEFLATED, 15, 8, st)
                assert b"".join(c.compress(r) for r in rows) + c.flush() == zlib_stream(b"".join(rows), level, st)


@pytest.mark.parametrize("interlace", [False, True])
@pytest.mark.parametrize("filter", sorted(FILTERS))
def test_pillow_decodes_to_the_input(filter, interlace):
    for bands in (1, 2, 3, 4):
        for h, w in ((1, 1), (3, 7), (9, 9), (33, 17), (64, 129)):
            for kind in ("noise", "photo"):
                a = frame(h, w, bands, seed=h * w + bands, kind=kind)
                png = vb.pngsave_host_twin(a, 6, filter=filter, interlace=interlace)
                assert np.array_equal(np.asarray(PIL.open(io.BytesIO(png))).reshape(h, w, bands), a), (bands, h, w, kind)
                if not interlace:   # the project's decoder loads non-interlaced streams: every filter type reversed
                    assert np.array_equal(vb.png_decode_host_twin(png), a), (bands, h, w, kind)


@pytest.mark.parametrize("opts", [dict(filter="paeth", interlace=True), dict(filter="up"), dict(interlace=True), dict(bitdepth=1),
                                  dict(bitdepth=2), dict(bitdepth=4)])
def test_stream_structure(opts):
    """IHDR carries the depth and interlace byte; the inflated scanlines start every row with the requested filter type"""
    for h, w in ((1, 1), (5, 3), (9, 9), (23, 41)):
        bands = 1 if "bitdepth" in opts else 3
        a = frame(h, w, bands, seed=h + w)
        cs = chunks(vb.pngsave_host_twin(a, **opts))
        depth, interlace = opts.get("bitdepth", 8), opts.get("interlace", False)
        assert cs[0][0] == b"IHDR" and struct.unpack(">IIBBBBB", cs[0][1]) == (w, h, depth, [0, 0, 4, 2, 6][bands], 0, 0, int(interlace))
        data = zlib.decompress(idat(vb.pngsave_host_twin(a, **opts)))
        at, types = 0, []
        for x0, y0, dx, dy in (ADAM7 if interlace else [(0, 0, 1, 1)]):
            pw, ph = max(0, -(-(w - x0) // dx)), max(0, -(-(h - y0) // dy))
            if pw and ph:
                for _ in range(ph):
                    types.append(data[at])
                    at += 1 + (pw * bands * depth + 7) // 8
        assert at == len(data) and types == [FILTERS[opts.get("filter", "none")]] * len(types)
        assert vb._png_scan_bytes(w, h, bands, interlace, depth) == len(data)


def test_defaults_unchanged():
    for bands in (1, 2, 3, 4):
        a = frame(31, 23, bands, kind="photo")
        base = vb.pngsave_host_twin(a, 7)
        assert vb.pngsave_host_twin(a, 7, filter="none", interlace=False, bitdepth=8) == base
        assert vb.pngsave_host_twin(a, 7, filter=0, bitdepth=0) == base
        assert vb.pngsave_host_twin(a, 7, filter=0x08) == base
        assert idat(base) == zlib_stream(b"".join(b"\0" + r.tobytes() for r in a), 7, zlib.Z_DEFAULT_STRATEGY)


DECLINES = [
    (dict(filter="all"), 3, "adaptive"),
    (dict(filter=0x30), 3, "more than one flag"),
    (dict(filter=0x90), 1, "more than one flag"),
    (dict(filter=0x01), 3, "unknown flag bits"),
    (dict(filter=0x108), 3, "unknown flag bits"),
    (dict(filter=-8), 3, "unknown flag bits"),
    (dict(bitdepth=16), 3, "bitdepth 16 is not built"),
    (dict(bitdepth=16), 1, "bitdepth 16 is not built"),
    (dict(bitdepth=3), 1, "bitdepth 3: PNG save takes"),
    (dict(bitdepth=12), 1, "bitdepth 12: PNG save takes"),
    (dict(bitdepth=4), 2, "no low-bit grey \\+ alpha"),
    (dict(bitdepth=2), 3, "quantisation is not built"),
    (dict(bitdepth=1), 4, "quantisation is not built"),
    (dict(bitdepth=1, filter="sub"), 1, "filter other than NONE or with interlace"),
    (dict(bitdepth=4, filter="paeth"), 1, "filter other than NONE or with interlace"),
    (dict(bitdepth=2, interlace=True), 1, "filter other than NONE or with interlace"),
]


@pytest.mark.parametrize("opts,bands,reason", DECLINES)
def test_declines(opts, bands, reason):
    """each decline is -1 with its reason from every entry point, before any device call"""
    a = np.zeros((3, 5, bands), np.uint8)
    with pytest.raises(vb.Error, match=reason):
        vb.pngsave_host_twin(a, **opts)
    with pytest.raises(vb.Error, match=reason):
        vb.pngsave_batch(a[None], **opts)
    with pytest.raises(vb.Error, match=reason):
        vb.Image(a).pngsave_buffer(**opts)


# ---------------------------------------------------------------------------------------------------------------- GPU

OPTION_SETS = [dict(filter=f, interlace=i) for f in sorted(FILTERS) for i in (False, True)]
LOW_BIT = [dict(bitdepth=d) for d in (1, 2, 4)]


@pytest.fixture(scope="module")
def gpu():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    vb.init(0)
    return torch


def device_out(src, where, frames_shape, opts, level=6):
    """vb200_pngsave_batch into device slots -> list of bytes"""
    torch = pytest.importorskip("torch")
    n, h, w, bands = frames_shape
    o = vb._png_options(level, "default", 1.0, opts.get("filter", "none"), opts.get("interlace", False), opts.get("bitdepth", 8))
    stride = vb._png_stride(w, h, bands, None, opts.get("interlace", False), opts.get("bitdepth", 8))
    dout = torch.zeros((n, stride), dtype=torch.uint8, device="cuda")
    lens = (C.c_size_t * n)()
    L = vb.lib()
    rc = L.vb200_pngsave_batch(src, where, w * bands, h * w * bands, n, w, h, bands, C.byref(o), None, 0, C.c_void_p(dout.data_ptr()), vb.DEVICE,
                               stride, lens)
    assert rc == 0, L.vb200_error_buffer()
    back = dout.cpu().numpy()
    return [back[i, :lens[i]].tobytes() for i in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("opts", OPTION_SETS + LOW_BIT, ids=lambda o: "-".join("%s=%s" % kv for kv in sorted(o.items())))
def test_device_equals_twin(gpu, opts):
    torch = gpu
    for bands in ((1,) if "bitdepth" in opts else (1, 2, 3, 4)):
        for h, w in ((1, 1), (7, 5), (33, 17), (64, 129)):
            frames = np.stack([frame(h, w, bands, seed=s, kind=("noise", "photo", "flat")[s % 3]) for s in range(4)])
            want = [vb.pngsave_host_twin(f, 6, **opts) for f in frames]
            assert vb.pngsave_batch(frames, 6, **opts) == want, (bands, h, w)
            t = torch.from_numpy(frames).cuda()
            assert vb.pngsave_batch(None, 6, in_ptr=t.data_ptr(), shape=frames.shape, **opts) == want, (bands, h, w)
            assert device_out(C.c_void_p(t.data_ptr()), vb.DEVICE, frames.shape, opts) == want, (bands, h, w)
            assert device_out(frames.ctypes.data_as(C.c_void_p), vb.HOST, frames.shape, opts) == want, (bands, h, w)


@pytest.mark.gpu
def test_device_small_budget_chunks(gpu):
    frames = np.stack([frame(40, 40, 4, seed=s, kind="photo") for s in range(9)])
    L = vb.lib()
    for opts in (dict(filter="paeth", interlace=True), dict(filter="avg")):
        try:
            L.vb200_debug_png_set_budget(1 << 20)
            got = vb.pngsave_batch(frames, 7, **opts)
        finally:
            L.vb200_debug_png_set_budget(0)
        assert got == [vb.pngsave_host_twin(f, 7, **opts) for f in frames], opts
    grey = np.stack([frame(40, 37, 1, seed=s, kind="photo") for s in range(9)])
    try:
        L.vb200_debug_png_set_budget(1 << 18)
        got = vb.pngsave_batch(grey, 7, bitdepth=4)
    finally:
        L.vb200_debug_png_set_budget(0)
    assert got == [vb.pngsave_host_twin(f, 7, bitdepth=4) for f in grey]


@pytest.mark.gpu
def test_device_tall_frame_and_many_tiles(gpu):
    tall = np.random.default_rng(4).integers(0, 3, (1, 70001, 3, 1), dtype=np.uint8)
    for opts in (dict(filter="paeth", interlace=True), dict(filter="up"), dict(bitdepth=2)):
        assert vb.pngsave_batch(tall, 6, **opts)[0] == vb.pngsave_host_twin(tall[0], 6, **opts), opts
    wide = np.stack([frame(500, 600, 3, seed=s, kind="photo") for s in range(2)])   # ~28 tiles of 32 KiB a frame
    for opts in (dict(filter="avg", interlace=True), dict(filter="sub")):
        got = vb.pngsave_batch(wide, 6, **opts)
        assert got == [vb.pngsave_host_twin(f, 6, **opts) for f in wide], opts


@pytest.mark.gpu
def test_device_buffer_equals_batch(gpu):
    for opts in OPTION_SETS[::3] + LOW_BIT:
        bands = 1 if "bitdepth" in opts else 4
        a = frame(45, 77, bands, seed=3, kind="photo")
        assert vb.Image(a).pngsave_buffer(5, "filtered", **opts) == vb.pngsave_batch(a[None], 5, "filtered", **opts)[0], opts


@pytest.mark.gpu
def test_png_thumbnail_resave_paeth_interlaced(gpu):
    from oracle import pyoracle
    srcs = [frame(200, 160, 4, seed=s, kind="photo") for s in range(3)]
    streams = []
    for s in srcs:
        buf = io.BytesIO()
        PIL.fromarray(s).save(buf, "PNG")
        streams.append(buf.getvalue())
    plan = vb.ThumbnailPlan(160, 200, 4, 64)
    th = plan.run_png(streams)
    got = vb.pngsave_batch(np.stack(th), 6, filter="paeth", interlace=True)
    for i in range(3):
        assert np.array_equal(th[i], pyoracle.thumbnail_image(srcs[i], 64))
        assert got[i] == vb.pngsave_host_twin(th[i], 6, filter="paeth", interlace=True)
        assert np.array_equal(np.asarray(PIL.open(io.BytesIO(got[i]))), th[i])


@pytest.mark.gpu
def test_low_bit_round_trip_through_the_device_decoder(gpu):
    for depth in (1, 2, 4):
        for w in (1, 2, 3, 8, 9, 17, 100):
            frames = np.stack([frame(13, w, 1, seed=s, kind="photo" if s else "noise") for s in range(3)])
            got = vb.png_decode_batch(vb.pngsave_batch(frames, 6, bitdepth=depth))
            for i in range(3):
                assert np.array_equal(got[i].reshape(13, w), low_bit_expected(frames[i], depth)), (depth, w, i)


@pytest.mark.gpu
def test_pool_after_decline_and_success(gpu):
    L = vb.lib()
    L.vb200_debug_dz_pool_used.restype = C.c_size_t
    frames = np.stack([frame(30, 30, 3, seed=s, kind="photo") for s in range(3)])
    vb.pngsave_batch(frames, 6, filter="paeth", interlace=True)
    pool = L.vb200_debug_dz_pool_used()
    with pytest.raises(vb.Error, match="quantisation"):
        vb.pngsave_batch(frames, 6, bitdepth=4)
    assert L.vb200_debug_dz_pool_used() == pool
    vb.pngsave_batch(frames, 6, filter="paeth", interlace=True)
    assert L.vb200_debug_dz_pool_used() == pool

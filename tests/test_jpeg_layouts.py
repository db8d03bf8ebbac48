"""JPEG decode of every chroma sampling layout the device path might meet, against libjpeg-turbo (csrc/jpeg.cu).

Pillow writes three layouts only (Y 1x1, 2x1 or 2x2 over Cb, Cr 1x1), so the streams here come from a small writer of
the test's own, built from ITU-T T.81: per-component sampling factors and quantisation tables, the Annex K Huffman
tables, restart intervals, baseline sequential and spectral-selection progressive frames.  Every stream goes to
libjpeg-turbo (inside Pillow) and to the decoder; each case must either give libjpeg-turbo's pixels bit for bit or be
declined with vb.Error -- never wrong pixels, and never a decode of a stream libjpeg-turbo refuses.
"""
import ctypes as C
import functools
import itertools
import os
import re

import numpy as np
import pytest

PIL = pytest.importorskip("PIL.Image")

# ------------------------------------------------------------------ a T.81 stream writer

# Figure A.6: zig-zag index -> row-major index within the 8x8 block
ZIGZAG = np.array(sorted(range(64), key=lambda n: (n // 8 + n % 8, n // 8 if (n // 8 + n % 8) % 2 else -(n // 8))))

# A.3.3: the FDCT as an orthonormal matrix product, F = D (f - 128) D^T
_u = np.arange(8)
DCT = np.sqrt(np.where(_u == 0, 1 / 8, 2 / 8))[:, None] * np.cos((2 * _u[None, :] + 1) * _u[:, None] * np.pi / 16)

# Tables K.1 / K.2 (row-major): luminance and chrominance quantisation
Q_LUMA = np.array([16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
                   14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
                   49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99])
Q_CHROMA = np.full(64, 99)
Q_CHROMA[[0, 1, 2, 3, 8, 9, 10, 11, 16, 17, 18, 24, 25]] = [17, 18, 24, 47, 18, 21, 26, 66, 24, 26, 56, 47, 66]

# Tables K.3 - K.6: (code counts by length 1..16, symbols).  The AC tables list their shorter codes' symbols; the 16-bit
# codes carry every remaining run / size symbol in increasing order.
_AC_SYMBOLS = [0x00, 0xF0] + [r << 4 | s for r in range(16) for s in range(1, 11)]


def _ac_table(counts, head):
    return counts, head + sorted(set(_AC_SYMBOLS) - set(head))


HUFF_DC = [([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12))),
           ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))]
HUFF_AC = [_ac_table([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 125],
                     [0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
                      0x32, 0x81, 0x91, 0xA1, 0x08, 0x23, 0x42, 0xB1, 0xC1, 0x15, 0x52, 0xD1, 0xF0, 0x24, 0x33, 0x62, 0x72, 0x82]),
           _ac_table([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 119],
                     [0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32,
                      0x81, 0x08, 0x14, 0x42, 0x91, 0xA1, 0xB1, 0xC1, 0x09, 0x23, 0x33, 0x52, 0xF0, 0x15, 0x62, 0x72, 0xD1, 0x0A, 0x16,
                      0x24, 0x34, 0xE1, 0x25, 0xF1])]


def _codes(table):
    """Annex C: symbol -> (code, length)"""
    counts, symbols = table
    out, code, k = {}, 0, 0
    for length, n in enumerate(counts, 1):
        for _ in range(n):
            out[symbols[k]] = (code, length)
            code, k = code + 1, k + 1
        code <<= 1
    return out


CODES_DC = [_codes(t) for t in HUFF_DC]
CODES_AC = [_codes(t) for t in HUFF_AC]


def _segment(marker, payload):
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + bytes(payload)


def _pack(codes, lengths):
    """the code words of one restart interval -> bytes: padded with 1-bits to a whole byte, a 00 stuffed after every FF"""
    if not codes:
        return b""
    n = np.asarray(lengths, np.int64)
    words = (np.asarray(codes, np.uint64) << (32 - n).astype(np.uint64)).astype(">u4")
    bits = np.unpackbits(words.view(np.uint8)).reshape(-1, 32)[np.arange(32) < n[:, None]]
    bits = np.concatenate([bits, np.ones(-len(bits) % 8, np.uint8)])
    return np.packbits(bits).tobytes().replace(b"\xff", b"\xff\x00")


class Frame:
    """The quantised coefficients of one frame: per component, zig-zag blocks over the MCU-padded block grid."""

    def __init__(self, planes, sampling, qscale=(50, 60, 80)):
        self.height, self.width = planes[0].shape
        self.sampling = list(sampling)
        hmax, vmax = max(h for h, _ in sampling), max(v for _, v in sampling)
        self.mcus_x = -(-self.width // (8 * hmax)) if len(sampling) > 1 else -(-self.width // 8)
        self.mcus_y = -(-self.height // (8 * vmax)) if len(sampling) > 1 else -(-self.height // 8)
        self.qt, self.coef, self.grid = [], [], []
        for c, (plane, (h, v)) in enumerate(zip(planes, sampling)):
            fx, fy = (hmax // h, vmax // v) if len(sampling) > 1 else (1, 1)
            cw, ch = -(-self.width * h // hmax), -(-self.height * v // vmax)   # A.1.1
            # box downsampling over the image replicated to whole boxes, then replication to the block grid
            p = np.pad(plane, ((0, ch * fy - self.height), (0, cw * fx - self.width)), mode="edge")
            p = p.reshape(ch, fy, cw, fx).mean(axis=(1, 3))
            bw, bh = (self.mcus_x * h, self.mcus_y * v) if len(sampling) > 1 else (self.mcus_x, self.mcus_y)
            p = np.pad(p, ((0, 8 * bh - ch), (0, 8 * bw - cw)), mode="edge")
            blocks = p.reshape(bh, 8, bw, 8).transpose(0, 2, 1, 3) - 128.0
            f = np.einsum("ux,byxk,vk->byuv", DCT, blocks, DCT).reshape(bh, bw, 64)
            q = np.clip((np.where(c, Q_CHROMA, Q_LUMA) * qscale[c] + 50) // 100, 2, 255)
            self.qt.append(q)
            self.coef.append(np.clip(np.rint(f / q), -1023, 1023).astype(np.int64)[..., ZIGZAG])
            self.grid.append((-(-ch // 8), -(-cw // 8)))    # the component's own blocks (A.2.2)

    def units(self, comps):
        """per unit (MCU) of a scan over `comps`: its blocks as (component, block row, block column)"""
        if len(comps) > 1:
            return [[(c, my * v + by, mx * h + bx) for c in comps for (h, v) in [self.sampling[c]] for by in range(v) for bx in range(h)]
                    for my in range(self.mcus_y) for mx in range(self.mcus_x)]
        (c,) = comps
        rows, cols = self.grid[c]
        return [[(c, by, bx)] for by in range(rows) for bx in range(cols)]


def _scan_data(frame, comps, ss, se, restart):
    """the entropy-coded segment of one scan (sequential when ss..se = 0..63, else a progressive first pass with Al = 0)"""
    intervals, codes, lengths = [], [], []
    units = frame.units(comps)
    for u, unit in enumerate(units):
        if u % (restart or len(units)) == 0:
            if u:
                intervals.append(_pack(codes, lengths))
                codes, lengths = [], []
            pred = {c: 0 for c in comps}
        for c, by, bx in unit:
            dc, ac = CODES_DC[min(c, 1)], CODES_AC[min(c, 1)]
            zz = frame.coef[c][by, bx]
            if ss == 0:
                diff = int(zz[0]) - pred[c]
                pred[c] = int(zz[0])
                s = abs(diff).bit_length()
                code, n = dc[s]
                codes.append(code << s | (diff if diff >= 0 else diff + (1 << s) - 1))
                lengths.append(n + s)
            if se == 0:
                continue
            band = zz[max(ss, 1):se + 1]
            last = max(ss, 1) - 1
            for k in np.flatnonzero(band) + max(ss, 1):
                run, val = int(k) - last - 1, int(zz[k])
                for _ in range(run // 16):
                    codes.append(ac[0xF0][0])
                    lengths.append(ac[0xF0][1])
                s = abs(val).bit_length()
                code, n = ac[(run % 16) << 4 | s]
                codes.append(code << s | (val if val >= 0 else val + (1 << s) - 1))
                lengths.append(n + s)
                last = int(k)
            if last < se:
                codes.append(ac[0x00][0])      # EOB (EOB0 in a progressive scan: a run of one block)
                lengths.append(ac[0x00][1])
    intervals.append(_pack(codes, lengths))
    return b"".join(seg + (bytes([0xFF, 0xD0 + i % 8]) if i + 1 < len(intervals) else b"") for i, seg in enumerate(intervals))


def write_jpeg(frame, mode="baseline", restart=0, jfif=True, ids=(1, 2, 3)):
    """mode: 'baseline' (one interleaved scan), 'separate' (sequential, one scan per component), 'progressive' (an
    interleaved DC scan, then AC bands per component) or 'progressive_dc_separate' (one DC scan per component)"""
    n = len(frame.sampling)
    out = b"\xff\xd8"
    if jfif:
        out += _segment(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for c in range(n):
        out += _segment(0xDB, [c] + [int(x) for x in frame.qt[c][ZIGZAG]])
    sof = [8, *frame.height.to_bytes(2, "big"), *frame.width.to_bytes(2, "big"), n]
    for c, (h, v) in enumerate(frame.sampling):
        sof += [ids[c], h << 4 | v, c]
    out += _segment(0xC2 if mode.startswith("progressive") else 0xC0, sof)
    dht = []
    for tc, tables in ((0, HUFF_DC), (1, HUFF_AC)):
        for th, (counts, symbols) in enumerate(tables):
            dht += [tc << 4 | th] + counts + symbols
    out += _segment(0xC4, dht)
    if restart:
        out += _segment(0xDD, restart.to_bytes(2, "big"))
    if mode == "baseline":
        scans = [(tuple(range(n)), 0, 63)]
    elif mode == "separate":
        scans = [((c,), 0, 63) for c in range(n)]
    else:
        dc = [tuple(range(n))] if mode == "progressive" else [(c,) for c in range(n)]
        bands = [[(1, 9), (10, 63)], [(1, 63)], [(1, 5), (6, 63)]]
        scans = [(comps, 0, 0) for comps in dc] + [((c,), ss, se) for c in range(n) for ss, se in bands[c]]
    for comps, ss, se in scans:
        sos = [len(comps)]
        for c in comps:
            t = min(c, 1)
            sos += [ids[c], (t << 4 | t) if se == 63 and ss == 0 else (t << 4 if ss == 0 else t)]
        out += _segment(0xDA, sos + [ss, se, 0]) + _scan_data(frame, comps, ss, se, restart)
    return out + b"\xff\xd9"


def ycc_planes(h, w, seed):
    """Y, Cb, Cr with structure in all three planes (chroma errors show) and noise (every coefficient position is used)"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = [128 + 90 * np.sin(xx / 9.0 + yy / 23.0), 128 + 80 * np.cos(xx / 13.0 - yy / 7.0), 128 + 70 * np.sin((xx * yy) / 150.0)]
    return [np.clip(b + rng.normal(0, 10, b.shape), 0, 255) for b in base]


# ------------------------------------------------------------------ the streams

from test_jpeg import turbo_decode  # noqa: E402

FACTORS = [(1, 1), (1, 2), (2, 1), (2, 2)]
LAYOUTS = list(itertools.product(FACTORS, repeat=3))    # (h, v) of Y, Cb, Cr
# (height, width): a multiple of every MCU, of none, one or two MCUs tall, one or two MCUs wide
SIZES = [(48, 64), (53, 37), (13, 130), (130, 11)]
# a restart interval of 7 MCUs divides no row of MCUs (nor of a component's blocks) at these sizes
VARIANTS = [("baseline", 0), ("baseline", 7), ("progressive", 0), ("progressive", 7)]
SHRINKS = (1, 2, 4, 8)

Y444, Y422, Y420 = ((1, 1), (1, 1), (1, 1)), ((2, 1), (1, 1), (1, 1)), ((2, 2), (1, 1), (1, 1))
U21, U12, U22 = ((2, 1),) * 3, ((1, 2),) * 3, ((2, 2),) * 3
Y22_C12 = ((2, 2), (1, 2), (1, 2))     # h2v1 chroma under a two-row MCU
Y440 = ((1, 2), (1, 1), (1, 1))        # h1v2 chroma: libjpeg's upsampler the device path does not have
PINNED = {Y444: "equal", Y422: "equal", Y420: "equal", U21: "equal", U12: "equal", Y22_C12: "equal",
          U22: "12 blocks per MCU", Y440: "needs an upsampler"}
# every reason the decoder gives for a layout it does not take
DECLINED = "needs an upsampler|blocks per MCU|unsupported sampling"


def layout_id(layout):
    return "_".join("%d%d" % f for f in layout)


@functools.cache
def frame(layout, size):
    h, w = size
    return Frame(ycc_planes(h, w, h * 131 + w), layout)


@functools.cache
def stream(layout, size, mode, restart, jfif=True, ids=(1, 2, 3)):
    return write_jpeg(frame(layout, size), mode, restart, jfif, ids)


@functools.cache
def libjpeg(data, shrink):
    """libjpeg-turbo's decode, or None where it refuses the stream"""
    try:
        return turbo_decode(data, shrink)
    except OSError:
        return None


def grey_stream(sampling, size, mode, restart):
    h, w = size
    return write_jpeg(Frame(ycc_planes(h, w, 7 + h + w)[:1], [sampling]), mode, restart)


def outcome(vb, data, shrink):
    """'equal' where the host twin gives libjpeg-turbo's pixels, the reason where it declines; fails on anything else"""
    want = libjpeg(data, shrink)
    try:
        got = vb.jpeg_decode_host_twin(data, shrink)
    except vb.Error as e:
        return str(e)
    assert want is not None, "decoded a stream libjpeg-turbo refuses"
    assert got.shape == want.shape, (got.shape, want.shape)
    bad = np.argwhere(got != want)
    assert not len(bad), "%d samples differ, first at %s: %d, libjpeg-turbo %d" % (len(bad), bad[0], got[tuple(bad[0])], want[tuple(bad[0])])
    return "equal"


@pytest.fixture(scope="module")
def vbl():
    import libvips_b200 as vb
    vb.lib()
    return vb


# ------------------------------------------------------------------ CPU: the host twin


def test_writer_codes_one_frame_in_every_scan_structure():
    """the writer's streams mean what they say: libjpeg-turbo decodes the interleaved sequential scan, one sequential scan
    per component and both progressive scan scripts of one frame to the same pixels, with and without restart markers"""
    for layout in (Y420, Y22_C12, ((1, 1), (2, 2), (1, 2))):
        for size in SIZES[:3]:
            want = libjpeg(stream(layout, size, "baseline", 0), 1)
            assert want is not None and want.shape == size + (3,)
            for mode in ("baseline", "separate", "progressive", "progressive_dc_separate"):
                for restart in (0, 7):
                    assert np.array_equal(libjpeg(stream(layout, size, mode, restart), 1), want), (layout, size, mode, restart)
    # and the pixels are the frame's: the decode of a 4:4:4 stream is close to the planes it was made from
    Y, Cb, Cr = ycc_planes(48, 64, 48 * 131 + 64)
    rgb = np.stack([Y + 1.402 * (Cr - 128), Y - 0.344136 * (Cb - 128) - 0.714136 * (Cr - 128), Y + 1.772 * (Cb - 128)], -1)
    assert np.abs(libjpeg(stream(Y444, (48, 64), "baseline", 0), 1) - np.clip(rgb, 0, 255)).mean() < 12


@pytest.mark.parametrize("layout", LAYOUTS, ids=layout_id)
def test_every_layout_matches_libjpeg_turbo_or_declines(vbl, layout):
    """all 64 three-component layouts with factors 1 or 2: baseline and spectral-selection progressive, with and without
    restart markers, at every shrink -- libjpeg-turbo's pixels, or a decline; PINNED layouts only the one or the other"""
    for size, (mode, restart), shrink in itertools.product(SIZES, VARIANTS, SHRINKS):
        data = stream(layout, size, mode, restart)
        try:
            got = outcome(vbl, data, shrink)
        except AssertionError as e:
            raise AssertionError("%s %s %s restart %d shrink %d: %s" % (layout_id(layout), size, mode, restart, shrink, e)) from None
        assert got == "equal" or re.search(DECLINED, got), got
        if layout in PINNED:
            assert re.search(PINNED[layout], got), (size, mode, restart, shrink, got)
    if layout == U22:
        assert libjpeg(stream(U22, SIZES[0], "baseline", 0), 1) is None     # libjpeg-turbo refuses it too


@pytest.mark.parametrize("sampling", [(2, 2), (1, 2), (2, 1)], ids=lambda s: "%dx%d" % s)
def test_greyscale_with_declared_sampling(vbl, sampling):
    """a one-component scan is never interleaved (T.81 A.2.2): whatever the frame header declares, one block per MCU"""
    for size, (mode, restart), shrink in itertools.product(SIZES, VARIANTS, SHRINKS):
        assert outcome(vbl, grey_stream(sampling, size, mode, restart), shrink) == "equal", (size, mode, restart, shrink)


def test_no_jfif_marker_and_other_component_ids(vbl):
    """without a JFIF marker libjpeg takes three components as YCbCr unless their ids are 'R' 'G' 'B'"""
    for layout in (Y420, U21, Y22_C12):
        for ids in ((0, 1, 2), (1, 2, 3), (7, 3, 250)):
            for mode, restart in VARIANTS[:3]:
                data = stream(layout, SIZES[1], mode, restart, jfif=False, ids=ids)
                for shrink in SHRINKS:
                    assert outcome(vbl, data, shrink) == "equal", (layout, ids, mode, restart, shrink)


def test_progressive_with_one_dc_scan_per_component(vbl):
    """the 10-block limit is on interleaved scans: 2x2 in every component decodes when no scan interleaves"""
    for layout in (U22, U21, Y420, ((1, 1), (2, 2), (1, 1))):
        for size in SIZES:
            for restart in (0, 7):
                data = stream(layout, size, "progressive_dc_separate", restart)
                for shrink in SHRINKS:
                    got = outcome(vbl, data, shrink)
                    assert got == "equal" or (layout not in (U22, U21, Y420) and re.search(DECLINED, got)), (layout, size, restart, shrink, got)


@pytest.mark.parametrize("layout", [((4, 1), (1, 1), (1, 1)), ((1, 3), (1, 1), (1, 1)), ((2, 1), (1, 3), (1, 3))], ids=layout_id)
def test_factors_beyond_two_are_declined(vbl, layout):
    """4:1:1 and vertical factors of 3: libjpeg-turbo decodes them (its integral upsampler), the device path declines"""
    for mode, restart in VARIANTS:
        data = stream(layout, SIZES[1], mode, restart)
        for shrink in SHRINKS:
            assert libjpeg(data, shrink) is not None
            with pytest.raises(vbl.Error, match=DECLINED):
                vbl.jpeg_decode_host_twin(data, shrink)


def test_one_sequential_scan_per_component_is_declined(vbl):
    for layout in (Y444, Y420, U12):
        for restart in (0, 7):
            data = stream(layout, SIZES[0], "separate", restart)
            assert np.array_equal(libjpeg(data, 2), libjpeg(stream(layout, SIZES[0], "baseline", restart), 2))
            for shrink in SHRINKS:
                with pytest.raises(vbl.Error, match="non-interleaved scans"):
                    vbl.jpeg_decode_host_twin(data, shrink)


# ------------------------------------------------------------------ GPU


def decodable(vb, data, shrink):
    """what the device path takes (its header checks run on the host: no GPU needed to ask)"""
    try:
        vb.jpeg_geometry([data], shrink)
        return True
    except vb.Error:
        return False


@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES, ids=lambda s: "%dx%d" % s)
def test_gpu_batches_of_mixed_layouts(vbl, size):
    """every layout the device path takes, baseline and progressive, with and without restart markers, in ONE batch per
    shrink: each frame carries its own sampling, DCT sizes, tables and path through the kernels"""
    import libvips_b200 as vb
    vb.init(0)
    for shrink in SHRINKS:
        streams = [stream(layout, size, mode, restart) for layout in LAYOUTS for mode, restart in VARIANTS]
        streams = [s for s in streams if decodable(vb, s, shrink)]
        assert len(streams) >= 4 * 8
        got = vb.jpeg_decode_batch(streams, shrink)
        for i, s in enumerate(streams):
            assert np.array_equal(got[i], libjpeg(s, shrink)), (size, shrink, i)
        grey = [grey_stream(f, size, mode, restart) for f in FACTORS for mode, restart in VARIANTS]
        assert np.array_equal(vb.jpeg_decode_batch(grey, shrink), np.stack([libjpeg(s, shrink) for s in grey])), (size, shrink)


@pytest.mark.gpu
def test_gpu_self_synchronising_decode_of_new_layouts(vbl):
    """scans without restart markers decoded by 128-byte subsequences (VB200_JPEG_SYNC), beside restart-interval frames"""
    import libvips_b200 as vb
    vb.init(0)
    layouts = (U21, U12, Y22_C12, Y420, ((1, 1), (2, 2), (1, 2)))
    os.environ["VB200_JPEG_SYNC"] = "128"
    try:
        for size in SIZES:
            fine = [Frame(ycc_planes(*size, seed), layout, qscale=(10, 15, 20)) for seed, layout in enumerate(layouts)]
            streams = [write_jpeg(f, "baseline", restart) for f in fine for restart in (0, 7)]
            # scans of 1 KB and more: eight subsequences or more each, so that they take the subsequence path
            assert all(len(s) - s.index(b"\xff\xda") > 1100 for s in streams[::2])
            for shrink in SHRINKS:
                batch = [s for s in streams if decodable(vb, s, shrink)]
                got = vb.jpeg_decode_batch(batch, shrink)
                for i, s in enumerate(batch):
                    assert np.array_equal(got[i], libjpeg(s, shrink)), (size, shrink, i)
    finally:
        del os.environ["VB200_JPEG_SYNC"]


@pytest.mark.gpu
def test_gpu_batch_with_a_declined_layout_fails_whole(vbl):
    """one frame the device path declines fails the batch before anything is decoded: no partial pixels"""
    import libvips_b200 as vb
    vb.init(0)
    good = [stream(layout, SIZES[0], "baseline", 7) for layout in (Y420, U21, U12)]
    for bad, shrink, reason in ((stream(U22, SIZES[0], "baseline", 0), 1, "12 blocks per MCU"),
                                (stream(U22, SIZES[0], "progressive", 7), 4, "12 blocks per MCU"),
                                (stream(Y440, SIZES[0], "baseline", 0), 1, "needs an upsampler"),
                                (stream(Y420, SIZES[0], "separate", 0), 2, "non-interleaved")):
        batch = vb.JpegBatch(good[:2] + [bad] + good[2:])
        with pytest.raises(vb.Error, match=reason):
            vb.jpeg_decode_batch(batch, shrink)
        h, w = SIZES[0][0] // shrink, SIZES[0][1] // shrink
        out = np.full((batch.n, h, w, 3), 0xA5, np.uint8)
        ww, hh, bb = C.c_int(), C.c_int(), C.c_int()
        with pytest.raises(vb.Error, match="frame 2: .*" + reason):
            vb._check(vb.lib().vb200_jpeg_decode_batch(batch.ptrs, batch.lens, batch.n, shrink, out.ctypes.data_as(C.c_void_p), vb.HOST,
                                                       w * 3, w * h * 3, C.byref(ww), C.byref(hh), C.byref(bb)))
        assert (out == 0xA5).all()
        # the same frames without it decode
        assert np.array_equal(vb.jpeg_decode_batch(good, shrink), np.stack([libjpeg(s, shrink) for s in good]))


@pytest.mark.gpu
def test_gpu_thumbnails_of_new_layouts(vbl):
    """vips_thumbnail_buffer's chain on uniform 2x1 and on Y 2x2 over chroma 1x2, at load-time shrinks 1, 2 and 4: the
    oracle thumbnail of libjpeg-turbo's decode"""
    import libvips_b200 as vb
    from oracle import pyoracle
    vb.init(0)
    for layout in (U21, Y22_C12):
        streams = [write_jpeg(Frame(ycc_planes(128, 120, seed), layout), mode, restart)
                   for seed, (mode, restart) in enumerate(VARIANTS)]
        for target in (40, 24, 12):
            shrink = vb.thumbnail_jpegshrink(120, 128, target)
            dw, dh, bands = vb.jpeg_geometry(streams, shrink)
            plan = vb.ThumbnailPlan(dw, dh, bands, target)
            got = plan.run_jpeg(streams, shrink)
            want = np.stack([pyoracle.thumbnail_image(libjpeg(s, shrink), target) for s in streams])
            assert got.shape == want.shape and np.array_equal(got, want), (layout_id(layout), target, shrink)
            for s, w in zip(streams, want):
                assert np.array_equal(vb.thumbnail_buffer(s, target), w), (layout_id(layout), target, shrink)
        assert {vb.thumbnail_jpegshrink(120, 128, t) for t in (40, 24, 12)} == {1, 2, 4}

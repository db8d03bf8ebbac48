"""Colour-managed thumbnails: vips_thumbnail's input_profile / output_profile / intent (resample/thumbnail.c:733-735,
929-970), the input-profile selection of vips_icc_set_import (colour/icc_transform.c:692-752) and the embedded JPEG profile
(foreign/jpeg2vips.c:699-799).

The expected output of each branch is the oracle thumbnail (pinned to the reference) followed by the ICC evaluator's host
twin (vb200_debug_icc_eval: mode 2 for the transform, mode 3 for the XYZ export), which the CPU tests hold to lcms2 through
oracle/pylcms.py at the bars of tests/test_icc.py; the GPU tests hold the device stage to that host-twin chain."""
import ctypes as C
import io
import os

import numpy as np
import pytest

import icc_fixtures as F
import libvips_b200 as vb
from oracle import pylcms

needs_lcms = pytest.mark.skipif(not pylcms.available(), reason="no lcms2 next to Pillow")
PROFILES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "profiles")


def P(name):
    with open(os.path.join(PROFILES, name), "rb") as f:
        return f.read()


SRGB, P3, GREY = P("sRGB.icm"), P("p3.icm"), P("sGrey.icm")
BUILTIN = {"srgb": SRGB, "sgrey": GREY}


def host_eval(mode, a, pa, pb=None):
    """the evaluator's per-pixel code on the CPU; a: (..., bands) uint8 -> (..., out bands) uint8"""
    L = vb.lib()
    a = np.ascontiguousarray(a, np.uint8)
    n = a.size // a.shape[-1]
    out = np.zeros((n, 8), np.uint8)
    ob = L.vb200_debug_icc_eval(mode, a.ctypes.data, 0, a.shape[-1], out.ctypes.data, n, pa, len(pa), pb, len(pb) if pb else 0, 1, 8, 0)
    if ob < 0:
        raise vb.Error(L.vb200_error_buffer().decode(errors="replace"))
    return np.ascontiguousarray(out.reshape(-1)[: n * ob].reshape(a.shape[:-1] + (ob,)))


def select(bands, embedded=None, input_profile=None, builtin=BUILTIN, intent="relative"):
    """(branch, source): ("T", "embedded" / "input" / "builtin") or ("X", None); raises vb.Error"""
    icc = vb.thumbnail_icc(SRGB, input_profile, intent, builtin)
    src = C.c_int()
    emb = bytes(embedded) if embedded else None
    rc = vb.lib().vb200_debug_icc_select(C.byref(icc), bands, emb, len(emb) if emb else 0, C.byref(src))
    if rc < 0:
        msg = vb.lib().vb200_error_buffer().decode(errors="replace")
        vb.lib().vb200_error_clear()
        raise vb.Error(msg)
    return ("X", None) if rc == 1 else ("T", ["embedded", "input", "builtin"][src.value])


def expected(thumb, out_profile, in_profile=None):
    """the host-twin chain after the oracle thumbnail: branch T with in_profile, branch X without"""
    return host_eval(2, thumb, in_profile, out_profile) if in_profile is not None else host_eval(3, thumb, out_profile)


# ------------------------------------------------------------------ embedded profile extraction

def _jpeg(a, **kw):
    from PIL import Image as PIL
    b = io.BytesIO()
    PIL.fromarray(a).save(b, "JPEG", quality=85, **kw)
    return b.getvalue()


def _app2(seq, count, payload, magic=b"ICC_PROFILE\0"):
    body = magic + bytes([seq, count]) + payload
    return b"\xff\xe2" + (len(body) + 2).to_bytes(2, "big") + body


def _insert_after_soi(stream, segments):
    return stream[:2] + b"".join(segments) + stream[2:]


def restated_profile(stream):
    """jpeg2vips.c:699-799 restated: APP2 segments before the first SOS, data_length > 14, "ICC_PROFILE" prefix, slot
    data[12] - 1 in 0..99 (later wins), concatenated up to the first empty slot"""
    slots, p = {}, 2
    while p < len(stream):
        while stream[p] != 0xFF:
            p += 1
        while stream[p] == 0xFF:
            p += 1
        m = stream[p]
        p += 1
        if m == 0xD8 or 0xD0 <= m <= 0xD7 or m == 0x01:
            continue
        L = int.from_bytes(stream[p:p + 2], "big")
        if m == 0xDA:
            break
        s = stream[p + 2:p + L]
        if m == 0xE2 and len(s) > 14 and s[:11] == b"ICC_PROFILE" and 0 <= s[12] - 1 < 100:
            slots[s[12] - 1] = s[14:]
        p += L
    out, k = b"", 0
    while k in slots:
        out += slots[k]
        k += 1
    return out or None


def test_embedded_profile_matches_pillow():
    from PIL import Image as PIL
    rng = np.random.default_rng(1)
    a = rng.integers(0, 256, (40, 56, 3), dtype=np.uint8)
    big2 = SRGB + bytes(rng.integers(0, 256, 70000 - len(SRGB), dtype=np.uint8))       # 2 chunks
    big3 = P3 + bytes(rng.integers(0, 256, 140000 - len(P3), dtype=np.uint8))          # 3 chunks
    for prof in (SRGB, P3, GREY, big2, big3):
        for kw in ({}, {"progressive": True}) if len(prof) < 65519 else ({},):     # Pillow's progressive writer buffers
            s = _jpeg(a if prof is not GREY else a[..., 0], icc_profile=prof, **kw)
            assert PIL.open(io.BytesIO(s)).info["icc_profile"] == prof
            assert vb.jpeg_icc_profile(s) == prof
    assert vb.jpeg_icc_profile(_jpeg(a)) is None
    with pytest.raises(vb.Error):
        vb.jpeg_icc_profile(b"not a jpeg")


def test_embedded_profile_chunk_rules():
    """hand-built APP2 sets against the restatement of jpeg2vips.c:699-799"""
    rng = np.random.default_rng(2)
    base = _jpeg(rng.integers(0, 256, (24, 24, 3), dtype=np.uint8))
    c = [bytes(rng.integers(0, 256, n, dtype=np.uint8)) for n in (300, 200, 100)]
    cases = {
        "in order": ([_app2(1, 3, c[0]), _app2(2, 3, c[1]), _app2(3, 3, c[2])], c[0] + c[1] + c[2]),
        "out of order": ([_app2(3, 3, c[2]), _app2(1, 3, c[0]), _app2(2, 3, c[1])], c[0] + c[1] + c[2]),
        "duplicate, last wins": ([_app2(1, 2, c[2]), _app2(2, 2, c[1]), _app2(1, 2, c[0])], c[0] + c[1]),
        "no first chunk": ([_app2(2, 3, c[1]), _app2(3, 3, c[2])], None),
        "gap truncates": ([_app2(1, 3, c[0]), _app2(3, 3, c[2])], c[0]),
        "seq 0 and 101 ignored": ([_app2(0, 1, c[1]), _app2(1, 1, c[0]), _app2(101, 1, c[2])], c[0]),
        "seq 100 kept, 255 ignored": ([_app2(1, 1, c[0]), _app2(100, 1, c[1]), _app2(255, 1, c[2])], c[0]),
        "count ignored": ([_app2(1, 9, c[0]), _app2(2, 0, c[1])], c[0] + c[1]),
        "other APP2": ([_app2(1, 1, c[0], magic=b"FPXR\0\0\0\0\0\0\0\0")], None),
    }
    for name, (segs, want) in cases.items():
        s = _insert_after_soi(base, segs)
        assert restated_profile(s) == want, name
        assert vb.jpeg_icc_profile(s) == want, name
    # segment lengths 13 .. 16: only data_length > 14 (a payload of 1+ byte after the 14-byte preamble) counts
    for dl in (13, 14, 15, 16):
        body = (b"ICC_PROFILE\0\x01\x01" + b"\x42\x43")[:dl]
        s = _insert_after_soi(base, [b"\xff\xe2" + (dl + 2).to_bytes(2, "big") + body])
        assert vb.jpeg_icc_profile(s) == restated_profile(s) == (body[14:] or None), dl
    # a chunk after the first SOS of a progressive stream is not read
    prog = _jpeg(rng.integers(0, 256, (32, 32, 3), dtype=np.uint8), progressive=True, icc_profile=c[0])
    second_sos = prog.index(b"\xff\xda", prog.index(b"\xff\xda") + 2)
    s = prog[:second_sos] + _app2(2, 2, c[1]) + prog[second_sos:]
    assert vb.jpeg_icc_profile(s) == restated_profile(s) == c[0]


# ------------------------------------------------------------------ input-profile selection

def test_selection_order():
    assert select(3, embedded=P3, input_profile=SRGB) == ("T", "embedded")
    assert select(3, input_profile=P3) == ("T", "input")
    assert select(3) == ("X", None)                                      # neither: vips_colourspace(XYZ) + export
    assert select(3, embedded=GREY, input_profile=P3) == ("T", "input")  # grey profile in an RGB frame: incompatible
    assert select(3, embedded=GREY) == ("T", "builtin")
    assert select(1, embedded=GREY) == ("T", "embedded")
    assert select(1, embedded=P3) == ("T", "builtin")
    assert select(3, embedded=P3[:100], input_profile=P3) == ("T", "input")   # truncated: lcms2 cannot open it
    assert select(4, embedded=SRGB) == ("T", "embedded")                   # RGBA: three colour bands
    with pytest.raises(vb.Error, match="built-in"):
        select(3, embedded=GREY, builtin={})
    with pytest.raises(vb.Error, match="frame 0"):
        select(3, embedded=GREY, builtin={"srgb": GREY})


def test_lut_profile_with_perceptual_intent_is_declined_not_skipped():
    """lcms2 would use the v4 lut RGB profile's A2B0 for the perceptual intent; the evaluator declines a lut profile at that
    intent (black point compensation), so the frame fails rather than falling through to input_profile.  A CMYK (ink)
    profile in an RGB frame is band-incompatible: that one is skipped"""
    ink = F.ink_profile()
    rgb_lut = F.lut_v4_rgb_profile("Lab ")
    assert vb.lib().vb200_debug_icc_classify(rgb_lut, len(rgb_lut), 3, 0) == 0      # lcms2 uses it for perceptual
    assert select(3, embedded=rgb_lut, input_profile=SRGB, intent="perceptual") == ("T", "embedded")
    with pytest.raises(vb.Error, match="intent"):
        host_eval_intent(np.zeros((1, 1, 3), np.uint8), rgb_lut, SRGB, 0)          # ... and the evaluator declines it
    assert vb.lib().vb200_debug_icc_classify(ink, len(ink), 3, 1) == 1              # CMYK in an RGB frame: skipped


def host_eval_intent(a, pa, pb, intent):
    L = vb.lib()
    out = np.zeros(8, np.uint8)
    if L.vb200_debug_icc_eval(2, a.ctypes.data, 0, 3, out.ctypes.data, 1, pa, len(pa), pb, len(pb), intent, 8, 0) < 0:
        raise vb.Error(L.vb200_error_buffer().decode(errors="replace"))
    return out


def _lcms_classify(prof, want_bands, intent):
    """vips_icc_load_profile_blob (icc_transform.c:581-652) asked of lcms2 itself"""
    L = pylcms.lib()
    L.cmsIsIntentSupported.argtypes = [C.c_void_p, C.c_uint, C.c_uint]
    L.cmsGetHeaderRenderingIntent.argtypes = [C.c_void_p]
    L.cmsGetHeaderRenderingIntent.restype = C.c_uint
    L.cmsGetColorSpace.argtypes = [C.c_void_p]
    L.cmsGetColorSpace.restype = C.c_uint
    h = L.cmsOpenProfileFromMem(prof, len(prof))
    if not h:
        return 1
    try:
        selected = intent
        if not L.cmsIsIntentSupported(h, intent, 0):
            hi = L.cmsGetHeaderRenderingIntent(h)
            if hi > 3:
                return 1
            selected = hi
        cs = L.cmsGetColorSpace(h).to_bytes(4, "big")
        bands = {b"GRAY": 1, b"RGB ": 3, b"Lab ": 3, b"XYZ ": 3, b"CMYK": 4, b"4CLR": 4}.get(cs, 0)
        if bands != want_bands or not L.cmsIsIntentSupported(h, selected, 0):
            return 1
        return 0 if selected == intent else 2
    finally:
        L.cmsCloseProfile(h)


def _mutants(rng, prof):
    prof = bytearray(prof)
    n_tags = int.from_bytes(prof[128:132], "big")
    out = [bytes(prof[:k]) for k in (0, 50, 127, 128, 131, 132, 140, 132 + 12 * n_tags - 1, len(prof) // 2)]
    def put(off, data):
        m = bytearray(prof)
        m[off:off + len(data)] = data
        out.append(bytes(m))
    put(36, b"acsq")
    for v in (b"\x02\x10", b"\x04\x40", b"\x05\x00", b"\x05\x01", b"\x06\x00", b"\x0a\x00", b"\x04\xff"):
        put(8, v)
    for cls in (b"scnr", b"prtr", b"link", b"abst", b"nmcl", b"xxxx", b"\0\0\0\0"):
        put(12, cls)
    for cs in (b"GRAY", b"CMYK", b"Lab ", b"HSV ", b"\0\0\0\0"):
        put(16, cs)
    for it in (0, 1, 2, 3, 4, 0x10000):
        put(64, it.to_bytes(4, "big"))
    for size in (0, 200, len(prof) - 1, len(prof) + 1000, 0xFFFFFFFF):
        put(0, size.to_bytes(4, "big"))
    for cnt in (0, 1, n_tags - 1, n_tags + 1, 100, 101, 0xFFFFFFFF):
        put(128, cnt.to_bytes(4, "big"))
    for i in range(n_tags):
        e = 132 + 12 * i
        put(e + 4, (0).to_bytes(4, "big"))                                    # offset 0: dropped
        put(e + 8, (0).to_bytes(4, "big"))                                    # size 0: dropped
        put(e + 4, (len(prof) - 4).to_bytes(4, "big"))                        # runs past the end: dropped
        put(e + 4, (0xFFFFFFF0).to_bytes(4, "big"))                           # wraps in 32 bits
        j = (i + 1) % n_tags
        put(e, bytes(prof[132 + 12 * j:132 + 12 * j + 4]))                   # duplicate signature
    for _ in range(60):
        m = bytearray(prof)
        for _ in range(int(rng.integers(1, 4))):
            m[int(rng.integers(0, 132 + 12 * n_tags))] ^= 1 << int(rng.integers(0, 8))
        out.append(bytes(m))
    return out


@needs_lcms
def test_classification_against_lcms2_mutants():
    """our open / compatibility / intent check never says "skip" where lcms2 would use the profile, nor the reverse"""
    rng = np.random.default_rng(3)
    n = 0
    for prof in (SRGB, P3, GREY, F.rgb_profile("srgb"), F.grey_profile(), F.ink_profile(), F.lut_v4_rgb_profile("Lab ")):
        for m in _mutants(rng, prof):
            for bands in (1, 3):
                for intent in (0, 1, 3):
                    got = vb.lib().vb200_debug_icc_classify(m, len(m), bands, intent)
                    assert got == _lcms_classify(m, bands, intent), (len(m), m[:20], bands, intent)
                    n += 1
    assert n > 3000


# ------------------------------------------------------------------ each branch against lcms2 (CPU)

def _frames(rng, shape):
    return rng.integers(0, 256, shape, dtype=np.uint8)


@needs_lcms
@pytest.mark.parametrize("pair", ["p3-srgb", "srgb-p3", "srgb-gamma", "table-srgb"])
def test_transform_branch_against_lcms2(oracle, pair):
    profs = {"p3": P3, "srgb": SRGB, "gamma": F.rgb_profile("gamma"), "table": F.rgb_profile("table")}
    pin, pout = (profs[k] for k in pair.split("-"))
    rng = np.random.default_rng(4)
    for bands in (3, 4):
        thumb = oracle.thumbnail_image(_frames(rng, (300, 420, bands)), 128)
        got = expected(thumb, pout, pin)
        want = pylcms.icc_transform(np.ascontiguousarray(thumb[..., :3]), pin, pout)
        d = np.abs(got[..., :3].astype(int) - want.astype(int))
        assert d.max() <= 1 and (d > 0).mean() < 0.03, (pair, d.max(), (d > 0).mean())
        if bands == 4:
            assert np.array_equal(got[..., 3], thumb[..., 3])                 # alpha rides along unchanged


@needs_lcms
@pytest.mark.parametrize("bands", [1, 2, 3, 4])
def test_export_branch_against_lcms2(oracle, bands):
    """no input profile: vips_colourspace(XYZ) (the oracle restates it) then vips_icc_export with the XYZ PCS"""
    rng = np.random.default_rng(5)
    thumb = oracle.thumbnail_image(_frames(rng, (260, 380, bands)), 100)
    src = "b-w" if bands < 3 else "srgb"
    xyz = oracle.colourspace(thumb, "xyz", src)
    for pout in (SRGB, P3, GREY):
        got = expected(thumb, pout)
        want = pylcms.icc_export(np.ascontiguousarray(xyz[..., :3]), pout, pcs="xyz")
        assert got.shape[-1] == want.shape[-1] + (bands - (1 if bands < 3 else 3))
        d = np.abs(got[..., :want.shape[-1]].astype(int) - want.astype(int))
        assert d.max() <= 1, (bands, d.max())
        if bands in (2, 4):
            assert np.array_equal(got[..., -1], np.clip(xyz[..., -1], 0, 255).astype(np.uint8))


# ------------------------------------------------------------------ the stored lcms2 fixture

def _fixture():
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import make_thumbnail_icc_golden as M
    return M, np.load(os.path.join(PROFILES, "..", "thumbnail_icc_lcms.npz"))


def within_lcms_bars(got, want, branch):
    """the CPU bars of tests/test_icc.py: a transform (lcms2's 1.14 fixed point) <= 1 LSB on < 3% of values; an export from
    float XYZ <= 1 LSB"""
    d = np.abs(got.astype(int) - want.astype(int))
    return d.max() <= 1 and (branch == "x" or (d > 0).mean() < 0.03)


@needs_lcms
def test_thumbnail_icc_fixture_is_current(oracle):
    """the stored thumbnails are the oracle's and the stored outputs lcms2's for the same inputs today (regenerate with
    make_thumbnail_icc_golden.py); the host twin of the stage meets the CPU bars against them"""
    M, G = _fixture()
    I = M.inputs()
    thumbs = {k: oracle.thumbnail_image(a, M.SIZE) for k, a in I.items()}
    now = M.lcms_outputs(oracle, thumbs)
    prof = M.profiles()
    for name, (bands, pin, pout) in M.CASES.items():
        assert np.array_equal(G["thumb_" + name], thumbs[name]), name
        assert np.array_equal(G["lcms_" + name], now[name]), name
        got = expected(thumbs[name], prof[pout], prof[pin] if pin else None)
        nc = now[name].shape[-1]
        assert within_lcms_bars(got[..., :nc], now[name], name[0]), name
        assert np.array_equal(got[..., nc:], thumbs[name][..., (1 if bands < 3 else 3):]), name


def test_other_interpretations_are_declined():
    """with a profile pair the reference keeps the image's interpretation and imports a CMYK image with its CMYK profile:
    the device stage takes sRGB / B_W frames only and says so, it does not treat C, M, Y as R, G, B"""
    a = np.zeros((16, 16, 4), np.uint8)
    with pytest.raises(vb.Error, match="interpretation"):
        vb.Image(a, "cmyk").thumbnail_image(8, output_profile=SRGB, embedded_profile=F.ink_profile(), builtin_profiles=BUILTIN)
    with pytest.raises(vb.Error, match="interpretation"):
        vb.Image(a[..., :3], "b-w").thumbnail_image(8, output_profile=SRGB)


# ------------------------------------------------------------------ plan interface without a GPU

def test_set_icc_refusals_need_no_pixels():
    """profiles are checked when set; a linear plan has no ICC stage"""
    with pytest.raises(vb.Error, match="linear"):
        vb.Image(np.zeros((8, 8, 3), np.uint8)).thumbnail_image(4, linear=True, output_profile=SRGB)


# ------------------------------------------------------------------ GPU

def _img(a):
    return vb.Image(a, "b-w" if a.shape[2] < 3 else "srgb")


def agree(got, want):
    d = np.abs(got.astype(int) - want.astype(int))
    return d.max() <= 1 and (d > 0).mean() < 1e-3


@pytest.mark.gpu
@pytest.mark.parametrize("bands", [1, 2, 3, 4])
def test_gpu_thumbnail_image_icc(vb, oracle, bands):
    rng = np.random.default_rng(10 + bands)
    a = _frames(rng, (333, 517, bands))
    thumb = oracle.thumbnail_image(a, 128)
    emb = GREY if bands < 3 else P3
    got = _img(a).thumbnail_image(128, output_profile=SRGB, embedded_profile=emb, builtin_profiles=BUILTIN).numpy()
    assert agree(got, expected(thumb, SRGB, emb))
    got = _img(a).thumbnail_image(128, output_profile=SRGB, builtin_profiles=BUILTIN).numpy()     # branch X
    assert agree(got, expected(thumb, SRGB))
    if bands in (2, 4):
        assert np.array_equal(got[..., -1], thumb[..., -1])
    # colour management off: the plain call's bytes
    assert np.array_equal(_img(a).thumbnail_image(128, output_profile=None, embedded_profile=emb).numpy(),
                          _img(a).thumbnail_image(128).numpy())


@pytest.mark.gpu
def test_gpu_output_bands_follow_the_profiles(vb, oracle):
    rng = np.random.default_rng(20)
    g = _frames(rng, (200, 300, 1))
    got = _img(g).thumbnail_image(64, output_profile=SRGB, embedded_profile=GREY).numpy()
    assert got.shape[-1] == 3 and agree(got, expected(oracle.thumbnail_image(g, 64), SRGB, GREY))
    ink = F.ink_profile()
    a = _frames(rng, (200, 300, 4))
    got = _img(a).thumbnail_image(64, output_profile=ink, embedded_profile=SRGB).numpy()
    want = expected(oracle.thumbnail_image(a, 64), ink, SRGB)
    assert got.shape[-1] == 5 and agree(got, want)


def _stream(a, prof=None, **kw):
    return _jpeg(a if a.shape[2] == 3 else a[..., 0], **({"icc_profile": prof} if prof else {}), **kw)


@pytest.mark.gpu
def test_gpu_run_jpeg_mixed_batch(vb, oracle):
    """P3, sRGB, untagged (branch X), grey-in-RGB (built-in fallback) and a 3-chunk profile in one batch: each frame equals
    the single-frame thumbnail_buffer result and its own branch's host-twin chain"""
    rng = np.random.default_rng(30)
    big = P3 + bytes(140000 - len(P3))                  # the header's size still says P3's: the rest is padding
    tags = [P3, SRGB, None, GREY, big, P3]
    streams = [_stream(_frames(rng, (256, 384, 3)), t) for t in tags]
    assert vb.jpeg_icc_profile(streams[4]) == big
    shrink = vb.thumbnail_jpegshrink(384, 256, 96)
    w, h, b = vb.jpeg_geometry(streams, shrink)
    plan = vb.ThumbnailPlan(w, h, b, 96)
    plan.set_icc(SRGB, builtin_profiles=BUILTIN)
    got = plan.run_jpeg(streams, shrink)
    dec = vb.jpeg_decode_batch(streams, shrink)
    inputs = [P3, SRGB, None, SRGB, big, P3]               # the grey profile does not fit an RGB frame: the built-in
    for i in range(len(tags)):
        single = vb.thumbnail_buffer(streams[i], 96, output_profile=SRGB, builtin_profiles=BUILTIN)
        assert np.array_equal(got[i], single), i
        assert agree(got[i], expected(oracle.thumbnail_image(dec[i], 96), SRGB, inputs[i])), i
    # the same plan with the stage off again: the plain bytes
    plan.set_icc(None)
    plain = vb.ThumbnailPlan(w, h, b, 96).run_jpeg(streams, shrink)
    assert np.array_equal(plan.run_jpeg(streams, shrink), plain)


@pytest.mark.gpu
@pytest.mark.parametrize("bands", [1, 2, 3, 4])
def test_gpu_plan_device_and_host(vb, oracle, bands):
    import torch
    rng = np.random.default_rng(40 + bands)
    n = 5
    frames = _frames(rng, (n, 240, 320, bands))
    plan = vb.ThumbnailPlan(320, 240, bands, 80)
    plain = plan.run_host(frames)
    emb = [P3, None, SRGB, P3, None] if bands >= 3 else [GREY, None, GREY, SRGB, None]
    plan.set_icc(P3 if bands >= 3 else SRGB, builtin_profiles=BUILTIN)
    out_profile = P3 if bands >= 3 else SRGB
    host = plan.run_host(frames, embedded=emb)
    din = torch.from_numpy(frames).cuda()
    dout = torch.empty((n, plan.out_height, plan.out_width, plan.out_bands), dtype=torch.uint8, device="cuda")
    plan.run_device(din.data_ptr(), dout.data_ptr(), n, embedded=emb)
    torch.cuda.synchronize()
    dev = dout.cpu().numpy()
    assert np.array_equal(host, dev)
    for i in range(n):
        inp = emb[i]
        if inp is not None and (inp is GREY) != (bands < 3):
            inp = GREY if bands < 3 else SRGB               # incompatible embedded profile: the built-in
        assert agree(dev[i], expected(plain[i], out_profile, inp)), i
    plan.set_icc(None)
    assert np.array_equal(plan.run_host(frames), plain)


@pytest.mark.gpu
def test_gpu_icc_then_sharpen(vb):
    import torch
    rng = np.random.default_rng(50)
    n = 3
    frames = torch.from_numpy(_frames(rng, (n, 300, 400, 4))).cuda()
    plan = vb.ThumbnailPlan(400, 300, 4, 100)
    plan.set_icc(SRGB, builtin_profiles=BUILTIN)
    emb = [P3] * n
    mid = torch.empty((n, plan.out_height, plan.out_width, 4), dtype=torch.uint8, device="cuda")
    plan.run_device(frames.data_ptr(), mid.data_ptr(), n, embedded=emb)
    want = torch.empty_like(mid)
    vb._check(vb.lib().vb200_sharpen_batch_device(C.c_void_p(mid.data_ptr()), mid[0].numel(), C.c_void_p(want.data_ptr()),
                                                  want[0].numel(), n, plan.out_width, plan.out_height, 4, 0.5, 2.0, 10.0, 20.0, 0.0, 3.0))
    plan.set_sharpen()
    got = torch.empty_like(mid)
    plan.run_device(frames.data_ptr(), got.data_ptr(), n, embedded=emb)
    torch.cuda.synchronize()
    assert torch.equal(got, want)


@pytest.mark.gpu
def test_gpu_70001_frames_one_call(vb):
    """more frames than one launch takes (32 768 a launch): the frame axis is chunked"""
    import torch
    n = 70001
    rng = np.random.default_rng(60)
    frames = _frames(rng, (n, 8, 8, 3))
    plan = vb.ThumbnailPlan(8, 8, 3, 4)
    plain = torch.empty((n, plan.out_height, plan.out_width, 3), dtype=torch.uint8, device="cuda")
    din = torch.from_numpy(frames).cuda()
    plan.run_device(din.data_ptr(), plain.data_ptr(), n)
    emb = [P3 if i % 3 == 0 else (SRGB if i % 3 == 1 else None) for i in range(n)]
    plan.set_icc(SRGB, builtin_profiles=BUILTIN)
    out = torch.empty_like(plain)
    plan.run_device(din.data_ptr(), out.data_ptr(), n, embedded=emb)
    torch.cuda.synchronize()
    p, o = plain.cpu().numpy(), out.cpu().numpy()
    for k, prof in ((0, P3), (1, SRGB), (2, None)):
        sel = np.arange(k, n, 3)
        assert agree(o[sel], expected(p[sel], SRGB, prof)), k


@pytest.mark.gpu
def test_gpu_against_lcms2_fixture(vb):
    """every device entry point on the seeded frames of thumbnail_icc_lcms.npz against lcms2's stored outputs, at the CPU
    bars: no lcms2 needed here, so a logic error shared by the kernel and its host twin cannot hide"""
    import torch
    M, G = _fixture()
    I = M.inputs()
    prof = M.profiles()
    for name, (bands, pin, pout) in M.CASES.items():
        want, thumb = G["lcms_" + name], G["thumb_" + name]
        nc, ec = want.shape[-1], (1 if bands < 3 else 3)
        emb = prof[pin] if pin else None
        a = I[name]
        img = _img(a).thumbnail_image(M.SIZE, output_profile=prof[pout], embedded_profile=emb, builtin_profiles=BUILTIN).numpy()
        plan = vb.ThumbnailPlan(a.shape[1], a.shape[0], bands, M.SIZE)
        plan.set_icc(prof[pout], builtin_profiles=BUILTIN)
        host = plan.run_host(a[None], embedded=[emb])[0]
        din = torch.from_numpy(np.ascontiguousarray(a[None])).cuda()
        dout = torch.empty((1, plan.out_height, plan.out_width, plan.out_bands), dtype=torch.uint8, device="cuda")
        plan.run_device(din.data_ptr(), dout.data_ptr(), 1, embedded=[emb])
        torch.cuda.synchronize()
        dev = dout.cpu().numpy()[0]
        for got in (img, host, dev):
            assert got.shape == want.shape[:-1] + (nc + bands - ec,), name
            assert within_lcms_bars(got[..., :nc], want, name[0]), name
            assert np.array_equal(got[..., nc:], thumb[..., ec:]), name        # alpha unchanged


@pytest.mark.gpu
def test_gpu_declined_profile_fails_the_batch_naming_the_frame(vb):
    """a profile lcms2 would use but the evaluator declines (a lut profile at the perceptual intent) fails the whole call"""
    import torch
    rgb_lut = F.lut_v4_rgb_profile("Lab ")
    plan = vb.ThumbnailPlan(64, 48, 3, 16)
    plan.set_icc(SRGB, intent="perceptual", builtin_profiles=BUILTIN)
    frames = torch.zeros((3, 48, 64, 3), dtype=torch.uint8, device="cuda")
    out = torch.empty((3, plan.out_height, plan.out_width, 3), dtype=torch.uint8, device="cuda")
    with pytest.raises(vb.Error, match="frame 1"):
        plan.run_device(frames.data_ptr(), out.data_ptr(), 3, embedded=[SRGB, rgb_lut, None])
    with pytest.raises(vb.Error, match="frame 1"):
        plan.run_host(frames.cpu().numpy(), embedded=[None, rgb_lut, SRGB])
    plan.run_device(frames.data_ptr(), out.data_ptr(), 3, embedded=[SRGB, P3, None])      # the plan still works


@pytest.mark.gpu
def test_gpu_linear_plan_refuses_icc(vb):
    plan = vb.ThumbnailPlan(256, 256, 3, 64, linear=True)
    icc = vb.thumbnail_icc(SRGB, builtin_profiles=BUILTIN)
    assert vb.lib().vb200_thumbnail_plan_set_icc(plan._p, C.byref(icc)) == -1
    assert "linear" in vb.lib().vb200_error_buffer().decode()
    vb.lib().vb200_error_clear()
    assert vb.lib().vb200_thumbnail_plan_output_bands(plan._p) == 3


@pytest.mark.gpu
def test_gpu_grey_jpeg(vb, oracle):
    """1-band JPEG streams through thumbnail_buffer_icc and run_jpeg: grey-tagged, untagged, and RGB-tagged (skipped for the
    built-in grey profile); grey output and RGB output"""
    rng = np.random.default_rng(70)
    tags = [GREY, None, SRGB]
    streams = [_stream(_frames(rng, (200, 280, 1)), t) for t in tags]
    shrink = vb.thumbnail_jpegshrink(280, 200, 64)
    w, h, b = vb.jpeg_geometry(streams, shrink)
    assert b == 1
    dec = vb.jpeg_decode_batch(streams, shrink)
    for out_profile in (GREY, SRGB):
        plan = vb.ThumbnailPlan(w, h, 1, 64)
        plan.set_icc(out_profile, builtin_profiles=BUILTIN)
        got = plan.run_jpeg(streams, shrink)
        assert got.shape[-1] == (1 if out_profile is GREY else 3)
        for i, t in enumerate(tags):
            single = vb.thumbnail_buffer(streams[i], 64, output_profile=out_profile, builtin_profiles=BUILTIN)
            assert np.array_equal(got[i], single), i
            inp = {0: GREY, 1: None, 2: GREY}[i]
            assert agree(got[i], expected(oracle.thumbnail_image(dec[i], 64), out_profile, inp)), i

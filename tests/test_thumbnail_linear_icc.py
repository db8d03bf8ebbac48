"""Colour-managed linear-light thumbnails: vips_thumbnail(..., linear = TRUE) with an embedded profile, input_profile and / or
output_profile (resample/thumbnail.c:766-805, 848-902, 929-987).

Per frame, one of three branches:
  I  a profile to import with (embedded, input_profile or the built-in sRGB one): vips_icc_import(XYZ) -> float premultiply
     (max_alpha 255) -> float resize -> unpremultiply (255) -> vips_icc_export to output_profile, or to the import's profile;
  X  only an output profile: the scRGB chain of the plain linear thumbnail, vips_colourspace(XYZ), vips_icc_export;
  plain: no profile anywhere, today's linear thumbnail.

The expected output of branch I / X is built from the oracle's float pieces (which the first test ties to the oracle's linear
thumbnail) around the ICC evaluator's host twin (vb200_debug_icc_eval modes 0 and 1); the CPU tests hold that chain to lcms2
(oracle/pylcms.py) at the ICC bars, and the GPU tests hold every device entry point to it."""
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
LUT = F.lut_v4_rgb_profile()


def drop_tags(prof, sigs):
    """the profile rebuilt without the tags named in sigs"""
    n = int.from_bytes(prof[128:132], "big")
    tags = []
    for i in range(n):
        e = 132 + 12 * i
        off, ln = int.from_bytes(prof[e + 4:e + 8], "big"), int.from_bytes(prof[e + 8:e + 12], "big")
        tags.append((prof[e:e + 4].decode("latin1"), prof[off:off + ln]))
    return F._profile(int.from_bytes(prof[8:12], "big"), prof[12:16].decode("latin1"), prof[16:20].decode("latin1"),
                      prof[20:24].decode("latin1"), [t for t in tags if t[0] not in sigs])


INPUT_ONLY = drop_tags(LUT, ("B2A0", "B2A1", "B2A2"))      # imports fine, cannot serve as an output profile


def ev(mode, a, pa, in_fmt=0, intent=1):
    """the evaluator's per-pixel code on the CPU, XYZ PCS: mode 0 uint8 -> float XYZ (+ float alpha), mode 1 float -> uint8"""
    L = vb.lib()
    a = np.ascontiguousarray(a)
    n = a.size // a.shape[-1]
    out = np.zeros((n, 8), np.float32 if mode == 0 else np.uint8)
    ob = L.vb200_debug_icc_eval(mode, a.ctypes.data, in_fmt, a.shape[-1], out.ctypes.data, n, pa, len(pa), None, 0, intent, 8, 1)
    if ob < 0:
        raise vb.Error(L.vb200_error_buffer().decode(errors="replace"))
    return np.ascontiguousarray(out.reshape(-1)[: n * ob].reshape(a.shape[:-1] + (ob,)))


def _geometry(oracle, a, target):
    hs, vs, _, _ = oracle.thumbnail_size(a.shape[1], a.shape[0], target)
    return hs, vs, a.shape[2] == 4 and hs != 1.0 and vs != 1.0


def float_chain(oracle, x, hs, vs, premul, max_alpha):
    """thumbnail.c:848-902 on a float image: premultiply, vips_resize, unpremultiply"""
    if premul:
        x = oracle.premultiply(x, max_alpha)
    x = oracle.resize(x, 1.0 / hs, 1.0 / vs)
    if premul:
        x = oracle.unpremultiply(x, max_alpha)
    return x


def scrgb_chain(oracle, a, target):
    hs, vs, premul = _geometry(oracle, a, target)
    return float_chain(oracle, oracle.colourspace(a, "scrgb", "srgb"), hs, vs, premul, 1.0)


def twin(oracle, a, target, pin=None, pout=None):
    """the expected frame: branch I with pin (export to pout, or to pin), branch X with pout only, plain with neither"""
    if pin is not None:
        hs, vs, premul = _geometry(oracle, a, target)
        x = float_chain(oracle, ev(0, a, pin), hs, vs, premul, 255.0)
        return ev(1, x, pout if pout is not None else pin, in_fmt=6)
    lin = scrgb_chain(oracle, a, target)
    if pout is None:
        return oracle.colourspace(lin, "srgb", "scrgb")
    return ev(1, oracle.colourspace(lin, "xyz", "scrgb"), pout, in_fmt=6)


def lcms_chain(oracle, a, target, pin=None, pout=None):
    """the same branches with lcms2 for the import and the export"""
    if pin is not None:
        hs, vs, premul = _geometry(oracle, a, target)
        x = pylcms.icc_import(np.ascontiguousarray(a[..., :3]), pin, pcs="xyz")
        if a.shape[2] == 4:
            x = np.concatenate([x, a[..., 3:].astype(np.float32)], -1)
        x = float_chain(oracle, x, hs, vs, premul, 255.0)
    else:
        x = oracle.colourspace(scrgb_chain(oracle, a, target), "xyz", "scrgb")
    out = pylcms.icc_export(np.ascontiguousarray(x[..., :3]), pout if pout is not None else pin, pcs="xyz")
    if a.shape[2] == 4:
        out = np.concatenate([out, np.clip(x[..., 3:], 0, 255).astype(np.uint8)], -1)
    return out


def within_lcms_bars(got, want, branch):
    """an export from float XYZ alone (branch X): <= 1 LSB, the bar of tests/test_thumbnail_icc.py.  With the import (branch I),
    lcms2 imports 8-bit codes through a prelinearised CLUT (its 8-bit -> 16-bit PCS optimisation) where the evaluator runs the
    profile's curves and matrix; the two differ by at most one 16-bit PCS step, which the float resize carries into the
    export.  The fractions measured per case are stored in thumbnail_linear_icc_lcms.npz (frac_*, written by
    make_thumbnail_linear_icc_golden.py, checked current below): 3.1-5.0% of values, each off by 1 LSB, the JPEG frames'
    small outputs at the top.  The bar: <= 1 LSB on < 6% of values.  The non-linear transform of tests/test_thumbnail_icc.py
    (one lcms2 transform, no float resize between import and export) stays under its 3%."""
    d = np.abs(got.astype(int) - want.astype(int))
    return d.max() <= 1 and (branch == "x" or (d > 0).mean() < 0.06)


def agree(got, want):
    d = np.abs(got.astype(int) - want.astype(int))
    return d.max() <= 1 and (d > 0).mean() < 1e-3


def _frames(rng, shape):
    return rng.integers(0, 256, shape, dtype=np.uint8)


# ------------------------------------------------------------------ CPU

@pytest.mark.parametrize("bands", [3, 4])
def test_composition_is_the_oracle_linear_thumbnail(oracle, bands):
    """the pieces the expected values are built from, with sRGB -> scRGB and max_alpha 1.0, are the pinned linear thumbnail"""
    rng = np.random.default_rng(100 + bands)
    for shape, target in (((300, 420), 128), ((256, 256), 64), ((333, 517), 100)):
        a = _frames(rng, shape + (bands,))
        assert np.array_equal(twin(oracle, a, target), oracle.thumbnail_image(a, target, linear=True)), shape


CASES = {  # name: (input profile or None, output profile or None)
    "p3-srgb": (P3, SRGB), "srgb-p3": (SRGB, P3), "gamma-srgb": (F.rgb_profile("gamma"), SRGB),
    "table-srgb": (F.rgb_profile("table"), SRGB), "lut-srgb": (LUT, SRGB), "p3-ink": (P3, F.ink_profile()),
    "p3-grey": (P3, GREY), "p3-none": (P3, None), "lut-none": (LUT, None), "x-srgb": (None, SRGB), "x-p3": (None, P3),
    "x-ink": (None, F.ink_profile()), "x-grey": (None, GREY),
}


@needs_lcms
@pytest.mark.parametrize("case", sorted(CASES))
def test_host_twin_chain_against_lcms2(oracle, case):
    pin, pout = CASES[case]
    rng = np.random.default_rng(200)
    for bands in (3, 4):
        a = _frames(rng, (240, 330, bands))
        got = twin(oracle, a, 90, pin, pout)
        want = lcms_chain(oracle, a, 90, pin, pout)
        assert got.shape == want.shape, (case, bands)
        nc = want.shape[-1] - (bands - 3)
        assert within_lcms_bars(got[..., :nc], want[..., :nc], "x" if pin is None else "i"), (case, bands)
        if bands == 4:
            assert np.array_equal(got[..., -1], want[..., -1]), case          # alpha survives the round trip


def lselect(bands, embedded=None, input_profile=None, output=SRGB, builtin=BUILTIN, intent="relative"):
    """(branch, source, export_from) of the stage's linear-mode choice; raises vb.Error"""
    icc = vb.linear_icc(output, input_profile, intent, builtin)
    b, s, e = C.c_int(), C.c_int(), C.c_int()
    emb = bytes(embedded) if embedded else None
    if vb.lib().vb200_debug_icc_select_linear(C.byref(icc), bands, emb, len(emb) if emb else 0, C.byref(b), C.byref(s), C.byref(e)):
        msg = vb.lib().vb200_error_buffer().decode(errors="replace")
        vb.lib().vb200_error_clear()
        raise vb.Error(msg)
    return b.value, s.value, e.value


def test_selection():
    I, X, PLAIN = 1, 2, 0
    assert lselect(3, P3) == (I, 0, 0)                                    # embedded usable
    assert lselect(4, P3, output=None) == (I, 0, 1)                       # ... and no output profile: export to it
    assert lselect(3, GREY, input_profile=P3) == (I, 1, 0)                # embedded unusable -> input_profile
    assert lselect(3, GREY, input_profile=P3, output=None) == (I, 1, 1)
    assert lselect(3, GREY) == (I, 2, 0)                                  # -> the built-in
    assert lselect(3, GREY, output=None) == (I, 2, 1)
    assert lselect(3, input_profile=SRGB, output=None) == (I, 1, 1)
    assert lselect(3) == (X, -1, 0)                                       # only an output profile
    assert lselect(3, output=None) == (PLAIN, -1, -1)                     # nothing: the plain path
    assert lselect(3, INPUT_ONLY) == (I, 0, 0)                            # imports fine, exports to output_profile
    with pytest.raises(vb.Error, match="no output profile"):
        lselect(3, INPUT_ONLY, output=None)                               # the reference's export fails
    with pytest.raises(vb.Error, match="built-in"):
        lselect(3, GREY, builtin={})


def test_refusals_need_no_pixels():
    """1- and 2-band frames (sGrey / GREY16 import) and other interpretations stay off the device; the profiles are checked
    before any pixel moves"""
    for a, interp in ((np.zeros((8, 8, 1), np.uint8), "b-w"), (np.zeros((8, 8, 2), np.uint8), "b-w"),
                      (np.zeros((8, 8, 4), np.uint8), "cmyk")):
        with pytest.raises(vb.Error, match="interpretation"):
            vb.Image(a, interp).thumbnail_image_linear(4, output_profile=SRGB, embedded_profile=F.ink_profile())
    a = np.zeros((8, 8, 3), np.uint8)
    with pytest.raises(vb.Error, match="corrupt"):
        vb.Image(a).thumbnail_image_linear(4, output_profile=SRGB[:100])
    with pytest.raises(vb.Error, match="rendering intent"):
        vb.Image(a).thumbnail_image_linear(4, output_profile=INPUT_ONLY)          # no B2A: not an output profile


# ------------------------------------------------------------------ the stored lcms2 fixture

def _fixture():
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import make_thumbnail_linear_icc_golden as M
    return M, np.load(os.path.join(PROFILES, "..", "thumbnail_linear_icc_lcms.npz"))


@needs_lcms
def test_linear_icc_fixture_is_current(oracle):
    """the stored lcms2 outputs, alpha bands, JPEG streams, decoded pixels and measured host-twin fractions are what the
    generator computes today (regenerate with make_thumbnail_linear_icc_golden.py); the host-twin chain meets the bars"""
    M, G = _fixture()
    now = M.build(oracle)
    assert sorted(now) == sorted(G.files)
    for k in now:
        assert np.array_equal(G[k], now[k]), k
    for name in list(M.CASES) + list(M.JPEG_CASES):
        assert float(G["frac_" + name]) < 0.06, name
    I = M.inputs()
    prof = M.profiles()
    for name, (bands, pin, pout) in M.CASES.items():
        want = G["lcms_" + name]
        got = twin(oracle, I[name], M.SIZE, prof[pin] if pin else None, prof[pout] if pout else None)
        assert within_lcms_bars(got[..., :want.shape[-1]], want, name[0]), name


# ------------------------------------------------------------------ GPU

def _img(a):
    return vb.Image(a, "srgb")


def _dev_run(plan, frames, embedded):
    import torch
    din = torch.from_numpy(np.ascontiguousarray(frames)).cuda()
    dout = torch.empty((len(frames), plan.out_height, plan.out_width, plan.out_bands), dtype=torch.uint8, device="cuda")
    plan.run_device(din.data_ptr(), dout.data_ptr(), len(frames), embedded=embedded)
    torch.cuda.synchronize()
    return dout.cpu().numpy()


def _jpeg(a, prof=None):
    from PIL import Image as PIL
    b = io.BytesIO()
    PIL.fromarray(a).save(b, "JPEG", quality=90, **({"icc_profile": prof} if prof else {}))
    return b.getvalue()


@pytest.mark.gpu
@pytest.mark.parametrize("bands", [3, 4])
def test_gpu_entry_points(vb, oracle, bands):
    """thumbnail_image_linear, plan device / host against the host-twin chain (and lcms2 where it is present) for each branch"""
    rng = np.random.default_rng(300 + bands)
    a = _frames(rng, (384, 512, bands))
    target = 64
    plan = vb.ThumbnailPlan(512, 384, bands, target, linear=True)
    assert plan.kernel == "linear_v_kernel + linear_h_kernel"
    for name in ("p3-srgb", "srgb-p3", "lut-srgb", "p3-none", "x-srgb", "x-p3"):
        pin, pout = CASES[name]
        want = twin(oracle, a, target, pin, pout)
        img = _img(a).thumbnail_image_linear(target, output_profile=pout, embedded_profile=pin, builtin_profiles=BUILTIN).numpy()
        plan.set_linear_icc(pout, builtin_profiles=BUILTIN)
        host = plan.run_host(a[None], embedded=[pin])[0]
        dev = _dev_run(plan, a[None], [pin])[0]
        for got in (img, host, dev):
            assert got.shape == want.shape and agree(got, want), name
        assert np.array_equal(img, dev) and np.array_equal(host, dev), name
        if pylcms.available():
            lc = lcms_chain(oracle, a, target, pin, pout)
            assert within_lcms_bars(dev[..., :3], lc[..., :3], "x" if pin is None else "i"), name


@pytest.mark.gpu
def test_gpu_jpeg_entry_points(vb, oracle):
    """thumbnail_buffer_linear decodes at full size and takes the stream's profile; run_jpeg (shrink 1) equals it"""
    rng = np.random.default_rng(310)
    tags = [P3, SRGB, None, GREY]
    streams = [_jpeg(_frames(rng, (256, 320, 3)), t) for t in tags]
    dec = vb.jpeg_decode_batch(streams, 1)
    plan = vb.ThumbnailPlan(320, 256, 3, 80, linear=True)
    for pout in (SRGB, None):
        plan.set_linear_icc(pout, builtin_profiles=BUILTIN)
        got = plan.run_jpeg(streams, 1)
        for i, t in enumerate(tags):
            single = vb.thumbnail_buffer_linear(streams[i], 80, output_profile=pout, builtin_profiles=BUILTIN)
            assert np.array_equal(got[i], single), (i, pout is None)
            pin = SRGB if t is GREY else t                          # a grey profile does not fit an RGB frame: the built-in
            assert agree(single, twin(oracle, dec[i], 80, pin, pout)), (i, pout is None)


@pytest.mark.gpu
def test_gpu_two_device_paths_agree(vb):
    """the two-kernel path equals the leaf chain, and linear_v2_kernel equals linear_v_kernel, byte for byte"""
    rng = np.random.default_rng(320)
    frames = _frames(rng, (4, 512, 512, 4))
    emb = [P3, LUT, None, SRGB]

    def run(env):
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            plan = vb.ThumbnailPlan(512, 512, 4, 64, linear=True)
        finally:
            for k, v in old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        plan.set_linear_icc(P3, builtin_profiles=BUILTIN)
        return plan, plan.run_host(frames, embedded=emb)

    fused, a = run({})
    assert fused.kernel == "linear_v_kernel + linear_h_kernel"
    leaf, b = run({"VB200_NO_LINEAR_FUSED": "1"})
    assert not leaf.fused
    static_off, c = run({"VB200_NO_LINEAR_STATIC": "1"})
    assert np.array_equal(a, b) and np.array_equal(a, c)


@pytest.mark.gpu
@pytest.mark.parametrize("bands", [3, 4])
def test_gpu_unchanged_where_nothing_is_managed(vb, bands):
    rng = np.random.default_rng(330 + bands)
    frames = _frames(rng, (3, 300, 400, bands))
    plan = vb.ThumbnailPlan(400, 300, bands, 100, linear=True)
    plain = plan.run_host(frames)
    plan.set_linear_icc(None, builtin_profiles=BUILTIN)                 # no output profile, untagged frames: today's bytes
    assert np.array_equal(plan.run_host(frames, embedded=[None] * 3), plain)
    assert np.array_equal(_img(frames[0]).thumbnail_image_linear(100).numpy(), _img(frames[0]).thumbnail_image(100, linear=True).numpy())
    plan.set_linear_icc(SRGB, builtin_profiles=BUILTIN)
    assert not np.array_equal(plan.run_host(frames, embedded=[P3] * 3), plain)
    plan.set_linear_icc(enabled=False)
    assert np.array_equal(plan.run_host(frames), plain)


@pytest.mark.gpu
def test_gpu_mixed_batch(vb, oracle):
    """P3, sRGB, untagged, grey-in-RGB (the built-in) and v4-lut frames in one batch: each equals its single-image call"""
    rng = np.random.default_rng(340)
    frames = _frames(rng, (5, 240, 320, 4))
    emb = [P3, SRGB, None, GREY, LUT]
    inputs = [P3, SRGB, None, SRGB, LUT]
    for pout in (SRGB, None):
        plan = vb.ThumbnailPlan(320, 240, 4, 80, linear=True)
        plan.set_linear_icc(pout, builtin_profiles=BUILTIN)
        got = plan.run_host(frames, embedded=emb)
        for i in range(5):
            single = _img(frames[i]).thumbnail_image_linear(80, output_profile=pout, embedded_profile=emb[i], builtin_profiles=BUILTIN).numpy()
            assert np.array_equal(got[i], single), (i, pout is None)
            want = twin(oracle, frames[i], 80, inputs[i], pout)
            assert agree(got[i], want), (i, pout is None)
            assert agree(got[i][..., 3], want[..., 3]), i                   # alpha


@pytest.mark.gpu
def test_gpu_band_changes_and_sharpen(vb, oracle):
    import torch
    rng = np.random.default_rng(350)
    a = _frames(rng, (256, 320, 4))
    ink = F.ink_profile()
    got = _img(a).thumbnail_image_linear(64, output_profile=ink, embedded_profile=P3).numpy()
    assert got.shape[-1] == 5 and agree(got, twin(oracle, a, 64, P3, ink))
    got = _img(a).thumbnail_image_linear(64, output_profile=GREY).numpy()
    assert got.shape[-1] == 2 and agree(got, twin(oracle, a, 64, None, GREY))
    # sharpen after a linear ICC batch
    n = 3
    frames = torch.from_numpy(_frames(rng, (n, 300, 400, 4))).cuda()
    plan = vb.ThumbnailPlan(400, 300, 4, 100, linear=True)
    plan.set_linear_icc(SRGB, builtin_profiles=BUILTIN)
    emb = [P3, None, LUT]
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
    """more frames than one launch takes (32 768): each frame's descriptor follows the chunk offset"""
    n = 70001
    rng = np.random.default_rng(360)
    base = _frames(rng, (3, 32, 32, 4))
    frames = np.ascontiguousarray(base[np.arange(n) % 3])
    emb = [(P3, SRGB, None)[i % 3] for i in range(n)]
    emb = [emb[i] if i % 3 != 1 else (SRGB if (i // 3) % 2 else LUT) for i in range(n)]
    plan = vb.ThumbnailPlan(32, 32, 4, 12, linear=True)
    assert plan.kernel == "linear_v_kernel + linear_h_kernel"
    plan.set_linear_icc(P3, builtin_profiles=BUILTIN)
    got = _dev_run(plan, frames, emb)
    for i in (0, 1, 2, 4, 32766, 32767, 32768, 32769, 32770, 65535, 65536, 65537, 69998, 69999, 70000):
        single = _img(frames[i]).thumbnail_image_linear(12, output_profile=P3, embedded_profile=emb[i], builtin_profiles=BUILTIN).numpy()
        assert np.array_equal(got[i], single), i


@pytest.mark.gpu
def test_gpu_declined_profile_and_refusals(vb):
    """a profile the evaluator declines (a lut profile at the perceptual intent) fails the batch naming its frame, and the plan
    still works; a non-linear plan and a corrupt output profile are refused when set"""
    import torch
    rgb_lut = F.lut_v4_rgb_profile("Lab ")
    plan = vb.ThumbnailPlan(64, 48, 3, 16, linear=True)
    plan.set_linear_icc(SRGB, intent="perceptual", builtin_profiles=BUILTIN)
    frames = torch.zeros((3, 48, 64, 3), dtype=torch.uint8, device="cuda")
    out = torch.empty((3, plan.out_height, plan.out_width, 3), dtype=torch.uint8, device="cuda")
    with pytest.raises(vb.Error, match="frame 1"):
        plan.run_device(frames.data_ptr(), out.data_ptr(), 3, embedded=[SRGB, rgb_lut, None])
    plan.run_device(frames.data_ptr(), out.data_ptr(), 3, embedded=[SRGB, P3, None])
    torch.cuda.synchronize()
    with pytest.raises(vb.Error, match="not linear"):
        vb.ThumbnailPlan(64, 48, 3, 16).set_linear_icc(SRGB)
    with pytest.raises(vb.Error, match="corrupt"):
        plan.set_linear_icc(SRGB[:100])
    with pytest.raises(vb.Error, match="no output profile"):
        plan.set_linear_icc(None)
        plan.run_host(frames.cpu().numpy(), embedded=[INPUT_ONLY, None, None])
    plan.set_linear_icc(SRGB)
    plan.run_host(frames.cpu().numpy(), embedded=[INPUT_ONLY, None, None])


def _fixture_cases(M, G):
    """(name, frame, input profile, output profile, lcms2 colour bands, alpha or None) of every stored case"""
    I, prof = M.inputs(), M.profiles()
    for name, (bands, pin, pout) in M.CASES.items():
        yield name, I[name], prof[pin] if pin else None, prof[pout] if pout else None, G["lcms_" + name], G.get("alpha_" + name)
    for name, (pin, pout) in M.JPEG_CASES.items():
        yield name, G["decoded_" + name], prof[pin], prof[pout] if pout else None, G["lcms_" + name], None


def _hold(got, want, alpha, name):
    nc = want.shape[-1]
    assert got.shape == want.shape[:-1] + (nc + (0 if alpha is None else 1),), name
    assert within_lcms_bars(got[..., :nc], want, name[0] if name[0] != "j" else "i"), name
    if alpha is not None:
        assert np.array_equal(got[..., nc:], alpha), name


@pytest.mark.gpu
def test_gpu_against_lcms2_fixture(vb):
    """every device entry point against lcms2's stored outputs at the CPU bars: no lcms2 needed here, so an error shared by
    the kernels and their host twin cannot hide"""
    M, G = _fixture()
    for name, a, pin, pout, want, alpha in _fixture_cases(M, G):
        img = _img(a).thumbnail_image_linear(M.SIZE, output_profile=pout, embedded_profile=pin, builtin_profiles=BUILTIN).numpy()
        plan = vb.ThumbnailPlan(a.shape[1], a.shape[0], a.shape[2], M.SIZE, linear=True)
        plan.set_linear_icc(pout, builtin_profiles=BUILTIN)
        host = plan.run_host(a[None], embedded=[pin])[0]
        dev = _dev_run(plan, a[None], [pin])[0]
        for got in (img, host, dev):
            _hold(got, want, alpha, name)
    for name, (pin, pout) in M.JPEG_CASES.items():
        stream = G["jpeg_" + name].tobytes()
        dec = G["decoded_" + name]
        assert np.array_equal(vb.jpeg_decode_batch([stream], 1)[0], dec), name
        pout = M.profiles()[pout] if pout else None
        buf = vb.thumbnail_buffer_linear(stream, M.SIZE, output_profile=pout, builtin_profiles=BUILTIN)
        plan = vb.ThumbnailPlan(dec.shape[1], dec.shape[0], 3, M.SIZE, linear=True)
        plan.set_linear_icc(pout, builtin_profiles=BUILTIN)
        jp = plan.run_jpeg([stream], 1)[0]
        for got in (buf, jp):
            _hold(got, G["lcms_" + name], None, name)


@pytest.mark.gpu
def test_gpu_odd_output_area_with_band_changes(vb):
    """a 4-band plan whose output frames are not a multiple of 4 bytes (5-band ink, 2-band grey + alpha over an odd OW x OH):
    the batch calls take the packed strides, each frame equals its single-image call"""
    rng = np.random.default_rng(370)
    frames = _frames(rng, (3, 512, 512, 4))
    emb = [P3, None, LUT]
    for pout, ob in ((F.ink_profile(), 5), (GREY, 2)):
        plan = vb.ThumbnailPlan(512, 512, 4, 63, linear=True)
        assert plan.out_width * plan.out_height % 2 == 1
        plan.set_linear_icc(pout, builtin_profiles=BUILTIN)
        assert plan.out_bands == ob
        host = plan.run_host(frames, embedded=emb)
        dev = _dev_run(plan, frames, emb)
        assert np.array_equal(host, dev)
        for i in range(3):
            single = _img(frames[i]).thumbnail_image_linear(63, output_profile=pout, embedded_profile=emb[i], builtin_profiles=BUILTIN).numpy()
            assert np.array_equal(dev[i], single), (ob, i)


@pytest.mark.gpu
def test_gpu_host_pump_names_the_batch_frame(vb):
    """the host pump runs 4K frames one slice at a time: a declined profile is still reported by its index in the batch"""
    rgb_lut = F.lut_v4_rgb_profile("Lab ")
    frames = np.zeros((3, 4096, 4096, 4), np.uint8)
    plan = vb.ThumbnailPlan(4096, 4096, 4, 512, linear=True)
    plan.set_linear_icc(SRGB, intent="perceptual", builtin_profiles=BUILTIN)
    with pytest.raises(vb.Error, match="frame 2"):
        plan.run_host(frames, embedded=[SRGB, None, rgb_lut])

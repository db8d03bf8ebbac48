"""Generate tests/golden/thumbnail_linear_icc_lcms.npz: lcms2's own outputs (the 2.18 inside Pillow, through oracle/pylcms.py,
which makes the reference's calls) for seeded colour-managed LINEAR thumbnails (thumbnail.c:766-805, 848-902, 929-987):
  - branch I, a profile to import with: vips_icc_import(pcs XYZ) by lcms2, the oracle's float premultiply (255) / resize /
    unpremultiply (255), vips_icc_export(XYZ PCS) by lcms2 to the output profile, or to the import's profile without one;
  - branch X, only an output profile: the oracle's scRGB linear chain, vips_colourspace(XYZ), vips_icc_export by lcms2.
Also stored per case: the alpha band the chain leaves, and the measured fraction of colour values where the ICC evaluator's
host twin (vb200_debug_icc_eval around the same oracle chain) differs from lcms2 -- the evidence behind the branch I bar in
tests/test_thumbnail_linear_icc.py.  The JPEG cases store the stream (Pillow-encoded, the profile in its APP2 segments) and
its decoded pixels (the decoder's host twin, pinned to libjpeg-turbo); they feed thumbnail_buffer_linear and run_jpeg.
tests/test_thumbnail_linear_icc.py holds every device entry point to these outputs, with neither lcms2 nor the reference at
run time.

    python tests/golden/make_thumbnail_linear_icc_golden.py
"""
import io
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import icc_fixtures as F  # noqa: E402
from oracle import pylcms  # noqa: E402

SIZE = 56
SHAPE = (160, 224)
JPEG_SHAPE = (96, 128)


def profiles():
    P = lambda n: open(os.path.join(HERE, "profiles", n), "rb").read()
    return {"srgb": P("sRGB.icm"), "p3": P("p3.icm"), "grey": P("sGrey.icm"), "lut": F.lut_v4_rgb_profile(), "ink": F.ink_profile()}


# name: (bands, input profile or None for branch X, output profile or None)
CASES = {
    "i_p3_srgb_rgba": (4, "p3", "srgb"),
    "i_srgb_p3_rgb": (3, "srgb", "p3"),
    "i_lut_srgb_rgba": (4, "lut", "srgb"),
    "i_p3_none_rgba": (4, "p3", None),
    "i_lut_none_rgb": (3, "lut", None),
    "i_p3_ink_rgba": (4, "p3", "ink"),
    "i_p3_grey_rgba": (4, "p3", "grey"),
    "x_srgb_rgba": (4, None, "srgb"),
    "x_p3_rgb": (3, None, "p3"),
    "x_ink_rgb": (3, None, "ink"),
    "x_grey_rgba": (4, None, "grey"),
}
# JPEG streams (3 bands): name: (embedded profile, output profile or None)
JPEG_CASES = {
    "j_p3_srgb": ("p3", "srgb"),
    "j_lut_none": ("lut", None),
    "j_srgb_p3": ("srgb", "p3"),
}


def inputs():
    """the seeded frames, shared with the tests: name -> uint8 (H, W, bands)"""
    rng = np.random.default_rng(2026)
    return {name: rng.integers(0, 256, SHAPE + (bands,), dtype=np.uint8) for name, (bands, _, _) in CASES.items()}


def jpeg_streams():
    """name -> the JPEG stream of a seeded smooth-ish RGB frame with the case's profile embedded"""
    from PIL import Image as PIL
    rng = np.random.default_rng(2027)
    prof = profiles()
    out = {}
    for name, (pin, _) in JPEG_CASES.items():
        a = np.clip(rng.normal(128, 60, JPEG_SHAPE + (3,)), 0, 255).astype(np.uint8)
        b = io.BytesIO()
        PIL.fromarray(a).save(b, "JPEG", quality=90, icc_profile=prof[pin])
        out[name] = b.getvalue()
    return out


def _chain_parts(oracle, a, pin):
    """the oracle's float chain: (float image before the export, branch)"""
    hs, vs, _, _ = oracle.thumbnail_size(a.shape[1], a.shape[0], SIZE)
    premul = a.shape[2] == 4 and hs != 1.0 and vs != 1.0

    def chain(x, max_alpha):
        if premul:
            x = oracle.premultiply(x, max_alpha)
        x = oracle.resize(x, 1.0 / hs, 1.0 / vs)
        return oracle.unpremultiply(x, max_alpha) if premul else x
    return chain, premul


def lcms_case(oracle, a, pin, pout):
    """(lcms2's colour bands, the chain's alpha band or None) for one frame"""
    chain, _ = _chain_parts(oracle, a, pin)
    if pin is not None:
        x = pylcms.icc_import(np.ascontiguousarray(a[..., :3]), pin, pcs="xyz")
        if a.shape[2] == 4:
            x = np.concatenate([x, a[..., 3:].astype(np.float32)], -1)
        x = chain(x, 255.0)
    else:
        x = oracle.colourspace(chain(oracle.colourspace(a, "scrgb", "srgb"), 1.0), "xyz", "scrgb")
    colour = pylcms.icc_export(np.ascontiguousarray(x[..., :3]), pout if pout is not None else pin, pcs="xyz")
    alpha = np.clip(x[..., 3:], 0, 255).astype(np.uint8) if a.shape[2] == 4 else None
    return colour, alpha


def twin_case(oracle, a, pin, pout):
    """the same chain around the ICC evaluator's host twin (vb200_debug_icc_eval, modes 0 and 1, XYZ PCS)"""
    import test_thumbnail_linear_icc as T
    return T.twin(oracle, a, SIZE, pin, pout)


def build(oracle):
    """everything the fixture stores, computed now"""
    prof = profiles()
    I = inputs()
    out = {}

    def put(name, a, pin, pout):
        pi, po = (prof[pin] if pin else None), (prof[pout] if pout else None)
        colour, alpha = lcms_case(oracle, a, pi, po)
        out["lcms_" + name] = colour
        if alpha is not None:
            out["alpha_" + name] = alpha
        got = twin_case(oracle, a, pi, po)[..., :colour.shape[-1]]
        out["frac_" + name] = np.array((got != colour).mean())
    for name, (bands, pin, pout) in CASES.items():
        put(name, I[name], pin, pout)
    import libvips_b200 as vb
    for name, s in jpeg_streams().items():
        out["jpeg_" + name] = np.frombuffer(s, np.uint8)
        dec = vb.jpeg_decode_host_twin(s)
        out["decoded_" + name] = dec
        put(name, dec, JPEG_CASES[name][0], JPEG_CASES[name][1])
    return out


def main():
    from oracle import pyoracle
    assert pylcms.available(), "no lcms2 next to Pillow"
    pyoracle.lib()
    out = build(pyoracle)
    path = os.path.join(HERE, "thumbnail_linear_icc_lcms.npz")
    np.savez_compressed(path, **out)
    print("wrote %s: %d cases, %d bytes" % (path, len(CASES) + len(JPEG_CASES), os.path.getsize(path)))
    for k in sorted(out):
        if k.startswith("frac_"):
            print("  %-22s host twin != lcms2 on %.4f of colour values" % (k[5:], float(out[k])))


if __name__ == "__main__":
    main()

"""Generate tests/golden/thumbnail_icc_lcms.npz: lcms2's own outputs (the 2.18 inside Pillow, through oracle/pylcms.py,
which makes the reference's calls) for seeded colour-managed thumbnails.  For each case the oracle thumbnail (pinned to
the reference) goes through what vips_thumbnail runs after the resize (thumbnail.c:929-970):
  - branch T, an input profile: vips_icc_transform, one lcms2 transform of the colour bands;
  - branch X, no input profile: vips_colourspace(XYZ) (the oracle restates it), then vips_icc_export with the XYZ PCS.
tests/test_thumbnail_icc.py compares the device stage with them, so the GPU suite holds an lcms2 comparison that needs
neither lcms2 nor the reference at run time.

    python tests/golden/make_thumbnail_icc_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))

import icc_fixtures as F  # noqa: E402
from oracle import pylcms  # noqa: E402

SIZE = 64


def profiles():
    P = lambda n: open(os.path.join(HERE, "profiles", n), "rb").read()
    return {"srgb": P("sRGB.icm"), "p3": P("p3.icm"), "grey": P("sGrey.icm"), "gamma": F.rgb_profile("gamma")}


# name: (bands, input profile or None for branch X, output profile)
CASES = {
    "t_p3_srgb_rgb": (3, "p3", "srgb"),
    "t_srgb_p3_rgba": (4, "srgb", "p3"),
    "t_gamma_srgb_rgb": (3, "gamma", "srgb"),
    "t_grey_srgb_bw": (1, "grey", "srgb"),
    "t_grey_grey_ga": (2, "grey", "grey"),
    "x_srgb_rgb": (3, None, "srgb"),
    "x_p3_rgba": (4, None, "p3"),
    "x_grey_bw": (1, None, "grey"),
    "x_srgb_ga": (2, None, "srgb"),
}


def inputs():
    """the seeded frames, shared with the tests: name -> uint8 (H, W, bands)"""
    rng = np.random.default_rng(2025)
    return {name: rng.integers(0, 256, (180, 260, bands), dtype=np.uint8) for name, (bands, _, _) in CASES.items()}


def lcms_outputs(oracle, thumbs):
    """name -> lcms2's colour bands for the case (the extra bands are the thumbnail's, checked separately)"""
    prof = profiles()
    out = {}
    for name, (bands, pin, pout) in CASES.items():
        t = thumbs[name]
        colour = 1 if bands < 3 else 3
        if pin is not None:
            out[name] = pylcms.icc_transform(np.ascontiguousarray(t[..., :colour]), prof[pin], prof[pout])
        else:
            xyz = oracle.colourspace(t, "xyz", "b-w" if bands < 3 else "srgb")
            out[name] = pylcms.icc_export(np.ascontiguousarray(xyz[..., :3]), prof[pout], pcs="xyz")
    return out


def main():
    from oracle import pyoracle
    assert pylcms.available(), "no lcms2 next to Pillow"
    I = inputs()
    thumbs = {name: pyoracle.thumbnail_image(a, SIZE) for name, a in I.items()}
    out = {"thumb_" + k: v for k, v in thumbs.items()}
    out.update({"lcms_" + k: v for k, v in lcms_outputs(pyoracle, thumbs).items()})
    path = os.path.join(HERE, "thumbnail_icc_lcms.npz")
    np.savez_compressed(path, **out)
    print("wrote %s: %d cases, %d bytes" % (path, len(CASES), os.path.getsize(path)))


if __name__ == "__main__":
    main()

"""vips_dzsave's strip walk for images with alpha: oracle/pydz.py's loop-for-loop restatement, with the shrink that
vips_region_shrink_method runs instead of region_shrink when vips_image_hasalpha holds (iofuncs/region.c:1551-1573):
vips_region_shrink_alpha (:1444-1482), restated here in double exactly as written there.

Everything else -- levels, strips, the odd-edge extras, tiles, the flush, the sidecar -- is pydz.Walk's own.
"""
import numpy as np

from oracle import pydz

# vips_interpretation_bands (iofuncs/image.c) for the Types a saved tile can have
INTERPRETATION_BANDS = {"b-w": 1, "srgb": 3, "multiband": 0}


def hasalpha(bands, interpretation):
    """vips_image_hasalpha, iofuncs/image.c:3113-3119: more bands than the Type has"""
    n = INTERPRETATION_BANDS[interpretation]
    return n > 0 and bands > n


def shrink_alpha(p00, p01, p10, p11):
    """SHRINK_ALPHA_TYPE(unsigned char), iofuncs/region.c:1446-1482, over arrays [..., bands] of the four pixels of each
    output pixel, in double as written there: alpha-weighted colour bands, alpha the mean alpha, 0 where it is 0; C's
    double-to-uchar conversion truncates"""
    a1, a2, a3, a4 = (p[..., -1].astype(np.float64) for p in (p00, p01, p10, p11))
    a = (a1 + a2 + a3 + a4) / 4.0
    out = np.zeros(p00.shape, np.uint8)
    nz = a != 0
    for z in range(p00.shape[-1] - 1):
        v = a1 * p00[..., z] + a2 * p01[..., z] + a3 * p10[..., z] + a4 * p11[..., z]
        out[..., z] = np.where(nz, np.trunc(v / np.where(nz, 4.0 * a, 1.0)), 0).astype(np.uint8)
    out[..., -1] = np.where(nz, np.trunc(a), 0).astype(np.uint8)
    return out


class Walk(pydz.Walk):
    """pydz.Walk whose shrink is vips_region_shrink_method's choice: the alpha shrink when the image has alpha"""

    def __init__(self, image, layout="dz", tile_size=None, overlap=None, depth=None, basename="untitled", suffix=None, interpretation=None):
        super().__init__(image, layout, tile_size, overlap, depth, basename, suffix)
        self.alpha = hasalpha(self.bands, interpretation or ("b-w" if self.bands < 3 else "srgb"))

    def region_shrink(self, src, dst, target):
        if not self.alpha:
            return super().region_shrink(src, dst, target)
        source = pydz.Rect(target.left * 2, target.top * 2, target.width * 2, target.height * 2)
        assert src.window(src.known, source).all(), "a shrink reads pixels nobody wrote"
        p = src.window(src.data, source)
        dst.window(dst.data, target)[...] = shrink_alpha(p[0::2, 0::2], p[0::2, 1::2], p[1::2, 0::2], p[1::2, 1::2])
        dst.window(dst.known, target)[...] = True


def dzsave(image, layout="dz", tile_size=None, overlap=None, depth=None, basename="untitled", suffix=None, strip_height=16, interpretation=None):
    """pydz.dzsave with the alpha-aware walk.  interpretation: "b-w", "srgb" or "multiband"; None is B_W below 3 bands and
    sRGB from 3, so 2 and 4 bands have alpha."""
    w = Walk(image, layout, tile_size, overlap, depth, basename, suffix, interpretation)
    height, width = w.image.shape[:2]
    for top in range(0, height, strip_height):
        w.pyramid_strip(pydz.Rect(0, top, width, min(strip_height, height - top)))
    return w

"""vips_dzsave's strip walk (libvips/foreign/dzsave.c), restated loop for loop in Python for the "dz" and "zoomify"
layouts, uchar pixels and region_shrink mean.

This is deliberately NOT the whole-image statement csrc/dzsave.cu runs ("each level is the 2 x 2 rounded mean of the level
above with its last column / row repeated when odd; tile (x, y) is a clipped rect of its level").  It keeps the
reference's machinery: a chain of levels each holding one strip of rows (pyramid_build :441-577), the image arriving in
strips of rows as vips_sink_disc hands them over (pyramid_strip :1942-2014), a strip that has filled writing its line of
tiles (strip_save / image_strip_allocate :1106-1152), filling its odd edges (level_generate_extras :1710-1754), shrinking
what it can into the strip below (strip_shrink :1761-1835 over vips_region_shrink_uncoded_mean, iofuncs/region.c:1139-1156),
moving down with the overlap rows carried across (strip_arrived :1845-1920), and the flush at the bottom (strip_flush
:1925-1937).  tests/test_dzsave.py holds the two statements against each other.

A region's buffer is new memory in the reference (vips_region_buffer, iofuncs/region.c:530-580, which also clips the rect
to the level's even-rounded image).  Here every region carries a mask of the pixels that have been written, and every read
-- a shrink, a tile -- asserts it reads written pixels only: the walk never depends on what a fresh buffer holds.
"""
import numpy as np


class Rect:
    def __init__(self, left, top, width, height):
        self.left, self.top, self.width, self.height = left, top, width, height

    @property
    def right(self):
        return self.left + self.width

    @property
    def bottom(self):
        return self.top + self.height

    def isempty(self):
        return self.width <= 0 or self.height <= 0

    def tuple(self):
        return (self.left, self.top, self.width, self.height)


def intersect(a, b):
    """vips_rect_intersectrect, iofuncs/rect.c: an empty result has width / height 0"""
    left, top = max(a.left, b.left), max(a.top, b.top)
    right, bottom = min(a.right, b.right), min(a.bottom, b.bottom)
    return Rect(left, top, max(0, right - left), max(0, bottom - top))


class Region:
    """a VipsRegion on a level's image (Xsize x Ysize), with a buffer"""

    def __init__(self, xsize, ysize, bands):
        self.xsize, self.ysize, self.bands = xsize, ysize, bands
        self.valid = Rect(0, 0, 0, 0)
        self.data = self.known = None

    def buffer(self, r):
        """vips_region_buffer: fresh memory for r clipped to the image"""
        c = intersect(r, Rect(0, 0, self.xsize, self.ysize))
        assert not c.isempty(), "valid clipped to nothing"
        self.valid = c
        self.data = np.full((c.height, c.width, self.bands), 0xA5, np.uint8)
        self.known = np.zeros((c.height, c.width), bool)

    def window(self, arr, r):
        y, x = r.top - self.valid.top, r.left - self.valid.left
        assert y >= 0 and x >= 0 and r.bottom <= self.valid.bottom and r.right <= self.valid.right, (r.tuple(), self.valid.tuple())
        return arr[y:y + r.height, x:x + r.width]


def region_copy(src, dst, r, x, y):
    """vips_region_copy(src, dst, r, x, y): rect r of src to (x, y) of dst"""
    d = Rect(x, y, r.width, r.height)
    pixels, known = src.window(src.data, r).copy(), src.window(src.known, r).copy()
    dst.window(dst.data, d)[...] = pixels
    dst.window(dst.known, d)[...] = known


class Level:
    pass


class Walk:
    def __init__(self, image, layout="dz", tile_size=None, overlap=None, depth=None, basename="untitled", suffix=None):
        a = np.ascontiguousarray(image, np.uint8)
        if a.ndim == 2:
            a = a[:, :, None]
        self.image = a
        self.bands = a.shape[2]
        self.layout = layout
        dz = layout == "dz"
        # vips_foreign_save_dz_build :2043-2113
        self.tile_size = tile_size if tile_size is not None else (254 if dz else 256)
        self.overlap = overlap if overlap is not None else (1 if dz else 0)
        self.suffix = suffix if suffix is not None else (".jpeg" if dz else ".jpg")
        if dz:
            self.tile_margin, self.tile_step = self.overlap, self.tile_size
        else:
            self.tile_margin, self.tile_step = 0, self.tile_size - self.overlap
        if self.tile_step <= 0:
            raise ValueError("overlap too large")
        self.depth = depth if depth is not None else ("onepixel" if dz else "onetile")
        self.imagename = basename
        self.root_name = basename + "_files" if dz else basename       # :2319-2322
        self.tile_count = 0
        self.tiles = []
        self.level = self.pyramid_build(None, a.shape[1], a.shape[0])

    # :441-577
    def pyramid_build(self, above, width, height):
        level = Level()
        level.width, level.height = width, height
        step = self.tile_step
        level.tiles_across = (width + step - 1) // step
        level.tiles_down = (height + step - 1) // step
        level.above, level.below = above, None
        level.xsize, level.ysize = width + (width & 1), height + (height & 1)
        level.strip = Region(level.xsize, level.ysize, self.bands)
        level.copy = Region(level.xsize, level.ysize, self.bands)
        level.y = level.write_y = 0
        h = self.tile_size + self.tile_margin
        if h & 1:
            h += 1
        level.strip.buffer(Rect(0, 0, level.xsize, h))
        limit = {"onepixel": 1, "onetile": self.tile_size, "one": max(width, height)}[self.depth]
        if width > limit or height > limit:
            level.below = self.pyramid_build(level, (width + 1) // 2, (height + 1) // 2)
            level.n = level.below.n + 1
        else:
            level.n = 0
        return level

    # :1156-1201
    def tile_name(self, level, x, y):
        if self.layout == "dz":
            return "%s/%d/%d_%d%s" % (self.root_name, level.n, x, y, self.suffix)
        n = 0
        p = level.below
        while p is not None:
            n += p.tiles_across * p.tiles_down
            p = p.below
        n += y * level.tiles_across + x
        self.tile_count += 1
        return "%s/TileGroup%d/%d-%d-%d%s" % (self.root_name, n // 256, level.n, x, y, self.suffix)

    # strip_save :1653-1703 with image_strip_allocate :1106-1152 and image_strip_work (the tile is the strip's pixels)
    def strip_save(self, level):
        x = 0
        image = Rect(0, 0, level.width, level.height)
        while x // self.tile_step < level.tiles_across:
            m = self.tile_margin
            pos = Rect(x - m, level.y - m, self.tile_size + 2 * m, self.tile_size + 2 * m)     # vips_rect_marginadjust
            pos = intersect(image, pos)
            assert not pos.isempty()
            assert level.strip.window(level.strip.known, pos).all(), ("a tile reads pixels nobody wrote", level.n, pos.tuple())
            pixels = level.strip.window(level.strip.data, pos).copy()
            tx, ty = x // self.tile_step, level.y // self.tile_step
            self.tiles.append((self.tile_name(level, tx, ty), level.n, tx, ty, pos.tuple(), pixels))
            x += self.tile_step

    # :1710-1754
    def level_generate_extras(self, level):
        strip = level.strip
        assert strip.valid.width == level.xsize
        if level.width < level.xsize:
            for arr in (strip.data, strip.known):
                arr[:, level.width] = arr[:, level.width - 1]
        if level.height < level.ysize:
            last = intersect(Rect(0, level.ysize - 2, level.xsize, 2), strip.valid)
            if last.height == 2:
                last.height = 1
                region_copy(strip, strip, last, 0, last.top + 1)

    # vips_region_shrink_method -> vips_region_shrink_uncoded_mean, iofuncs/region.c:1139-1156, 1250-1290
    def region_shrink(self, src, dst, target):
        source = Rect(target.left * 2, target.top * 2, target.width * 2, target.height * 2)
        assert src.window(src.known, source).all(), "a shrink reads pixels nobody wrote"
        p = src.window(src.data, source).astype(np.int32)
        tot = p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2]
        dst.window(dst.data, target)[...] = ((tot + 2) >> 2).astype(np.uint8)
        dst.window(dst.known, target)[...] = True

    # :1761-1835
    def strip_shrink(self, level):
        below = level.below
        src, to = level.strip, below.strip
        self.level_generate_extras(level)
        while True:
            target = intersect(Rect(0, below.write_y, below.xsize, to.valid.height), to.valid)
            source = Rect(target.left * 2, target.top * 2, target.width * 2, target.height * 2)
            source = intersect(source, src.valid)
            target = Rect(source.left // 2, source.top // 2, source.width // 2, source.height // 2)
            if target.isempty():
                break
            self.region_shrink(src, to, target)
            below.write_y += target.height
            if below.write_y == to.valid.bottom or below.write_y == below.height:
                self.strip_arrived(below)

    # :1845-1920
    def strip_arrived(self, level):
        self.strip_save(level)
        if level.below is not None:
            self.strip_shrink(level)
        level.y += self.tile_step
        new_strip = Rect(0, level.y - self.tile_margin, level.xsize, self.tile_size + 2 * self.tile_margin)
        new_strip = intersect(new_strip, Rect(0, 0, level.xsize, level.ysize))
        if new_strip.height & 1:
            new_strip.height += 1
        if new_strip.bottom == level.height:
            new_strip.height = level.ysize - new_strip.top
        overlap = intersect(new_strip, level.strip.valid)
        if not overlap.isempty():
            level.copy.buffer(overlap)
            region_copy(level.strip, level.copy, overlap, overlap.left, overlap.top)
        if not new_strip.isempty():
            level.strip.buffer(new_strip)
            if not overlap.isempty():
                region_copy(level.copy, level.strip, overlap, overlap.left, overlap.top)

    # :1925-1937
    def strip_flush(self, level):
        if level.y < level.height:
            self.strip_save(level)
        if level.below is not None:
            self.strip_flush(level.below)

    # :1942-2014: one strip of the image from vips_sink_disc
    def pyramid_strip(self, area):
        level = self.level
        region = Region(self.image.shape[1], self.image.shape[0], self.bands)
        region.valid = area
        region.data = self.image[area.top:area.bottom]
        region.known = np.ones(region.data.shape[:2], bool)
        while True:
            to = level.strip.valid
            target = intersect(Rect(0, level.write_y, level.xsize, to.height), to)
            target = intersect(target, area)
            if target.isempty():
                break
            region_copy(region, level.strip, target, target.left, target.top)
            level.write_y += target.height
            if level.write_y == to.bottom or level.write_y == level.height:
                self.strip_arrived(level)
        if level.write_y == level.height:
            self.strip_flush(level)

    # write_dzi :579-620, write_properties :622-655
    def sidecar(self):
        if self.layout == "dz":
            text = ('<?xml version="1.0" encoding="UTF-8"?>\n'
                    '<Image xmlns="http://schemas.microsoft.com/deepzoom/2008"\n'
                    '  Format="%s"\n  Overlap="%d"\n  TileSize="%d"\n  >\n  <Size \n    Height="%d"\n    Width="%d"\n  />\n</Image>\n'
                    % (self.suffix[1:], self.overlap, self.tile_size, self.level.height, self.level.width))
            return self.imagename + ".dzi", text
        text = ('<IMAGE_PROPERTIES WIDTH="%d" HEIGHT="%d" NUMTILES="%d" NUMIMAGES="1" VERSION="1.8" TILESIZE="%d" />\n'
                % (self.level.width, self.level.height, self.tile_count, self.tile_size))
        return self.root_name + "/ImageProperties.xml", text

    def levels(self):
        out, p = [], self.level
        while p is not None:
            out.append((p.n, p.width, p.height, p.tiles_across, p.tiles_down))
            p = p.below
        return sorted(out)


def dzsave(image, layout="dz", tile_size=None, overlap=None, depth=None, basename="untitled", suffix=None, strip_height=16):
    """Run the walk over `image` (H x W or H x W x bands uint8) fed in strips of strip_height rows (vips_sink_disc hands over
    16 at a time; the result must not depend on it).  Returns the Walk: .tiles = [(name, n, x, y, (left, top, width, height),
    pixels)] in the order written, .levels(), .sidecar()."""
    w = Walk(image, layout, tile_size, overlap, depth, basename, suffix)
    height, width = w.image.shape[:2]
    for top in range(0, height, strip_height):
        w.pyramid_strip(Rect(0, top, width, min(strip_height, height - top)))
    return w

"""Every template instantiation of the three fused thumbnail kernels, bit for bit against the oracle.

thumbnail_fused.cu runs an 8-bit RGBA thumbnail plan on one of three kernels, each a family of template instantiations:

- thumbnail_fused_mma_kernel<VS, NP, PREMUL, HS, OPQ> (v4, reducev on the tensor pipe): one per VB200_V4_LIST key
  (VS, NP, HS), each compiled premultiplied with the opaque-stage vote off, premultiplied with it on, and plain;
- thumbnail_fused_tma_kernel<VS, NP, PREMUL> (v2): VS 1, 2, 3, 4, 8 or 0 (any other box, read at run time), NP 0, 6 or 7;
- thumbnail_fused_kernel<VS, PREMUL> (v1, ld.global): VS 1, 2, 3, 4, 5, 6, 8 or 0.

The CPU half pins, through the host-only hook vb200_debug_thumbnail_kernel, a plan for every instantiation a plan can
reach, in both alpha modes, and checks that the table covers the lists above.  The GPU half runs every row against the
oracle, bit for bit:

- at two frame scales: a small frame (one band CTA) and a wide one (at least three bands, the last one shorter, and
  where the kernel allows it a last box cut short on both axes);
- as one frame per batch, where rows_per_cta splits the rows over CTAs, and as a batch large enough that every CTA
  takes whole frames;
- on random RGBA, alpha exactly 0, 1, 254 and 255, constant 0 and 255, impulses on a lattice, the band seams and the
  last row and column, and horizontal and vertical ramps;
- for v4: with the opaque-stage vote forced on and off over a batch that mixes opaque and live-alpha frames, with the
  row-by-row stage copy in place of the tensor map (VB200_NO_TENSORMAP), and through vb200_thumbnail_batch_device with a
  base pointer 4 bytes off the 16-byte grid, which runs v1 on the same plan.

The GPU half's 120 cases take about 65 s on one H100 80GB HBM3 (700 W power limit), most of it host copies and the oracle.
"""
import ctypes as C
import math
import re

import numpy as np
import pytest

import libvips_b200 as vb

SIZES = {"both": 0, "force": 3}

# the instantiations of thumbnail_fused_mma_kernel (VB200_V4_LIST in thumbnail_fused.cu)
V4_LIST = [(4, 6, 4), (4, 7, 4), (2, 6, 2), (2, 7, 2), (8, 6, 8), (8, 7, 8),
           (4, 0, 4), (2, 0, 2), (4, 0, 2), (2, 0, 4), (4, 0, 8), (2, 0, 8), (8, 0, 8), (8, 0, 4),
           (3, 0, 3), (5, 0, 5), (6, 0, 6), (7, 0, 7), (2, 0, 3), (3, 0, 2), (3, 0, 4), (4, 0, 3),
           (4, 0, 5), (5, 0, 4), (5, 0, 6), (6, 0, 5), (6, 0, 7), (7, 0, 6), (7, 0, 8), (8, 0, 7)]
# the boxes the switches of launch_tma_vs and launch_ldg_vs instantiate (0: any other box), and v2's NP (launch_tma)
V2_VS, V2_NP = (1, 2, 3, 4, 8, 0), (0, 6, 7)
V1_VS = (1, 2, 3, 4, 5, 6, 8, 0)
# v2 at box 8 is compiled but no plan reaches it: its stage ring alone (3 stages x 2 x 8 rows x 2336 bytes = 112 128)
# leaves 3 584 bytes of v2's 113 KiB shared-memory bound, less than its pair slots, output rows and tables take, so such
# a plan runs v4 or v1.  test_v2_box_8_is_unreachable is the search that shows it.
V2_UNREACHABLE = {(8, 0), (8, 6), (8, 7)}

# (W, H, target_w, target_h, size) of a small frame and of a wide one, per instantiation; each runs premultiplied and plain.
# The small frames are the smallest the search over frames up to 256 x 256 found with both sides of the output >= 6.  The
# wide frames have more output rows than one CTA takes from a lone frame (33 for v4, 17 for v1 and v2); for v4, H % VS != 0, and W % HS != 0 where HS is 3, 5, 6 or 7
# (a v4 frame is a whole number of 16-byte units, and the plan gives box 8 to v1 when its last box is cut short).
V4_GEOM = {
    (2, 0, 2): ((28, 31, 7, None, "both"), (2232, 161, 513, 40, "force")),
    (2, 0, 3): ((40, 24, 6, 6, "force"), (1372, 203, 228, None, "both")),
    (2, 0, 4): ((48, 35, 6, 8, "force"), (4104, 161, 513, 40, "force")),
    (2, 0, 8): ((192, 30, 12, 7, "force"), (8208, 161, 513, 40, "force")),
    (2, 6, 2): ((28, 31, 7, 6, "force"), (1500, 161, 375, None, "both")),
    (2, 7, 2): ((36, 51, 12, None, "both"), (1492, 161, 363, None, "both")),
    (3, 0, 2): ((28, 47, 7, 7, "force"), (2052, 241, 513, 40, "force")),
    (3, 0, 3): ((36, 51, 8, None, "both"), (1372, 199, 228, None, "both")),
    (3, 0, 4): ((60, 43, 7, 7, "force"), (1452, 262, 181, None, "both")),
    (4, 0, 2): ((36, 51, 9, 6, "force"), (2052, 321, 513, 40, "force")),
    (4, 0, 3): ((36, 51, 6, 6, "force"), (1348, 321, 170, None, "both")),
    (4, 0, 4): ((88, 48, 10, 6, "force"), (1424, 321, 163, None, "both")),
    (4, 0, 5): ((88, 48, 8, 6, "force"), (1324, 339, 131, None, "both")),
    (4, 0, 8): ((136, 49, 8, 6, "force"), (8208, 321, 513, 40, "force")),
    (4, 6, 4): ((88, 48, 11, None, "both"), (1464, 321, 183, None, "both")),
    (4, 7, 4): ((48, 95, 11, None, "both"), (1440, 321, 173, None, "both")),
    (5, 0, 4): ((48, 95, 6, 9, "force"), (1436, 401, 145, None, "both")),
    (5, 0, 5): ((60, 87, 8, None, "both"), (1304, 401, 119, None, "both")),
    (5, 0, 6): ((84, 63, 7, 6, "force"), (1304, 467, 108, None, "both")),
    (6, 0, 5): ((60, 87, 6, 7, "force"), (1308, 481, 110, None, "both")),
    (6, 0, 6): ((84, 74, 7, None, "both"), (1276, 481, 97, None, "both")),
    (6, 0, 7): ((84, 74, 6, 6, "force"), (7704, 521, 531, 40, "force")),
    (7, 0, 6): ((80, 84, 6, None, "both"), (1280, 561, 92, None, "both")),
    (7, 0, 7): ((92, 93, 6, None, "both"), (1152, 561, 75, None, "both")),
    (7, 0, 8): ((96, 87, 6, 6, "force"), (8800, 601, 517, 40, "force")),
    (8, 0, 4): ((48, 96, 6, 6, "force"), (4104, 641, 513, 40, "force")),
    (8, 0, 7): ((100, 97, 7, 6, "force"), (1156, 641, 73, None, "both")),
    (8, 0, 8): ((176, 97, 10, None, "both"), (1312, 641, 75, None, "both")),
    (8, 6, 8): ((96, 118, 6, 7, "force"), (1392, 641, 87, None, "both")),
    (8, 7, 8): ((96, 118, 7, None, "both"), (1344, 641, 81, None, "both")),
}
# v2, (VS as named, NP): VS "0(b)" is the run-time form at box b.  Boxes 6 and 7 with NP 7 have no wide frame: the search
# over outputs 130 wide found none (the v2 plan's threads and shared memory grow with the band; such plans run v1).
V2_GEOM = {
    ("1", 0): ((16, 16, 6, None, "both"), (260, 32, 208, 25, "force")),
    ("1", 6): ((16, 16, 8, None, "both"), (260, 38, 173, 25, "force")),
    ("1", 7): ((60, 43, 7, 21, "force"), (552, 55, 129, 27, "force")),
    ("2", 0): ((20, 33, 10, 8, "force"), (260, 98, 208, 24, "force")),
    ("2", 6): ((16, 45, 8, 11, "force"), (276, 100, 157, 25, "force")),
    ("2", 7): ((76, 46, 7, 11, "force"), (1304, 103, 130, 25, "force")),
    ("3", 0): ((16, 45, 8, 7, "force"), (260, 146, 208, 24, "force")),
    ("3", 6): ((16, 73, 8, 12, "force"), (264, 150, 150, 25, "force")),
    ("3", 7): ((88, 45, 7, 7, "force"), (1304, 152, 130, 25, "force")),
    ("4", 0): ((16, 68, 8, 8, "force"), (260, 194, 208, 24, "force")),
    ("4", 6): ((16, 73, 8, 9, "force"), (260, 194, 173, 24, "force")),
    ("4", 7): ((92, 93, 6, 11, "force"), (1564, 203, 130, 25, "force")),
    ("0(5)", 0): ((16, 68, 8, 6, "force"), (260, 242, 208, 24, "force")),
    ("0(5)", 6): ((16, 91, 8, 9, "force"), (260, 242, 173, 24, "force")),
    ("0(5)", 7): ((52, 94, 12, 9, "force"), (552, 247, 129, 24, "force")),
    ("0(6)", 0): ((16, 73, 6, 6, "force"), (260, 290, 208, 24, "force")),
    ("0(6)", 6): ((16, 73, 8, 6, "force"), (260, 290, 173, 24, "force")),
    ("0(6)", 7): ((60, 87, 7, 7, "force"), None),
    ("0(7)", 0): ((16, 91, 8, 6, "force"), (260, 338, 208, 24, "force")),
    ("0(7)", 6): ((60, 87, 30, 6, "force"), (260, 338, 173, 24, "force")),
    ("0(7)", 7): ((60, 89, 7, 6, "force"), None),
}
# v1: frames whose rows are not a whole number of 16-byte units
V1_GEOM = {
    "1": ((29, 18, 14, None, "both"), (261, 33, 208, 26, "force")),
    "2": ((22, 35, 11, 8, "force"), (261, 99, 208, 24, "force")),
    "3": ((21, 39, 10, 6, "force"), (261, 147, 208, 24, "force")),
    "4": ((23, 54, 11, 6, "force"), (261, 195, 208, 24, "force")),
    "5": ((18, 71, 9, 7, "force"), (261, 243, 208, 24, "force")),
    "6": ((18, 79, 9, 6, "force"), (261, 291, 208, 24, "force")),
    "8": ((17, 125, 8, 7, "force"), (261, 387, 208, 24, "force")),
    "0(9)": ((16, 109, 8, 6, "force"), (261, 435, 208, 24, "force")),
    "0(13)": ((147, 183, 7, None, "both"), (261, 627, 208, 24, "force")),
}


def v4_name(key, alpha):
    return "thumbnail_fused_mma_kernel<VS=%d,NP=%d,%s,HS=%d,cols=768,cpt=2>" % (key[0], key[1], alpha, key[2])


def v2_name(key, alpha):
    return "thumbnail_fused_tma_kernel<VS=%s,NP=%d,%s>" % (key[0], key[1], alpha)


def v1_name(key, alpha):
    return "thumbnail_fused_kernel<VS=%s,%s>" % (key, alpha)


# (family, key, has_alpha, small geometry, wide geometry, kernel name)
CASES = [(fam, key, alpha, small, wide, namer(key, "premul" if alpha else "plain"))
         for fam, table, namer in (("v4", V4_GEOM, v4_name), ("v2", V2_GEOM, v2_name), ("v1", V1_GEOM, v1_name))
         for key, (small, wide) in table.items()
         for alpha in (True, False)]


def case_id(c):
    return "%s-%s-%s" % (c[0], "-".join(str(k) for k in c[1]) if isinstance(c[1], tuple) else c[1], "premul" if c[2] else "plain")


def _lib():
    L = C.CDLL(vb.library_path())
    L.vb200_debug_thumbnail_kernel.argtypes = [C.c_int] * 7 + [C.c_char_p, C.c_int]
    L.vb200_debug_thumbnail_pages_size.argtypes = [C.c_int] * 6 + [C.POINTER(C.c_double)] * 2 + [C.POINTER(C.c_int)] * 3
    L.vb200_debug_thumbnail_bands.argtypes = [C.c_int] * 3 + [C.POINTER(C.c_int)] * 7 + [C.c_int] + [C.POINTER(C.c_int)] * 2
    return L


def kernel_name(geom, alpha):
    w, h, tw, th, size = geom
    buf = C.create_string_buffer(160)
    assert _lib().vb200_debug_thumbnail_kernel(w, h, 4, int(alpha), tw, th or 0, SIZES[size], buf, len(buf)) == 0, geom
    return buf.value.decode()


def out_size(geom):
    w, h, tw, th, size = geom
    hs, vs = C.c_double(), C.c_double()
    ow, oh, ph = C.c_int(), C.c_int(), C.c_int()
    assert _lib().vb200_debug_thumbnail_pages_size(w, h, 1, tw, th or tw, SIZES[size], C.byref(hs), C.byref(vs), C.byref(ow),
                                                    C.byref(oh), C.byref(ph)) == 0, geom
    return ow.value, oh.value


def v4_bands(geom):
    """The tensor-pipe kernel's bands of a square-target "both" plan: [(xa, xb, c_lo, c_hi)], the last band's reach (its
    c_lo plus the width of its TMA boxes), or None for any other plan"""
    w, h, tw, th, size = geom
    if size != "both" or th is not None:
        return None
    cap = 64
    xa, xb, c_lo, c_hi, seam = [(C.c_int * cap)() for _ in range(5)]
    ow, nb, boxw, nbox = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    rc = _lib().vb200_debug_thumbnail_bands(w, h, tw, C.byref(ow), C.byref(nb), xa, xb, c_lo, c_hi, seam, cap, C.byref(boxw),
                                            C.byref(nbox))
    if rc:
        return None
    n = nb.value
    return [(xa[i], xb[i], c_lo[i], c_hi[i]) for i in range(n)], c_lo[n - 1] + nbox.value * boxw.value


# ------------------------------------------------------------------ CPU: the table names what it claims

@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_case_names_its_instantiation(case):
    fam, key, alpha, small, wide, want = case
    assert kernel_name(small, alpha) == want, small
    if wide is not None:
        assert kernel_name(wide, alpha) == want, wide


def test_cases_cover_every_instantiation():
    """Every v4 key, every v2 (VS, NP) but the unreachable ones and every v1 VS, premultiplied and plain"""
    got = {"v4": set(), "v2": set(), "v1": set()}
    for fam, key, alpha, small, wide, name in CASES:
        m = re.fullmatch(r"thumbnail_fused_mma_kernel<VS=(\d+),NP=(\d+),(\w+),HS=(\d+),cols=768,cpt=2>", name)
        if m:
            got["v4"].add((int(m[1]), int(m[2]), int(m[4]), m[3]))
            continue
        m = re.fullmatch(r"thumbnail_fused_tma_kernel<VS=(\d+)(?:\(\d+\))?,NP=(\d+),(\w+)>", name)
        if m:
            got["v2"].add((int(m[1]), int(m[2]), m[3]))
            continue
        m = re.fullmatch(r"thumbnail_fused_kernel<VS=(\d+)(?:\(\d+\))?,(\w+)>", name)
        assert m, name
        got["v1"].add((int(m[1]), m[2]))
    alphas = ("premul", "plain")
    assert got["v4"] == {k + (a,) for k in V4_LIST for a in alphas}
    assert got["v2"] == {(vs, np_, a) for vs in V2_VS for np_ in V2_NP for a in alphas if (vs, np_) not in V2_UNREACHABLE}
    assert got["v1"] == {(vs, a) for vs in V1_VS for a in alphas}


def test_run_time_box_is_named_as_such():
    """A box the v1 / v2 switch does not list runs the VS = 0 instantiation, and the name says so"""
    assert kernel_name((4096, 4096, 150, None, "both"), True) == "thumbnail_fused_kernel<VS=0(13),premul>"
    assert kernel_name((16, 68, 8, 6, "force"), True) == "thumbnail_fused_tma_kernel<VS=0(5),NP=0,premul>"
    assert kernel_name((18, 71, 9, 7, "force"), True) == "thumbnail_fused_kernel<VS=5,premul>"


def test_v2_box_8_is_unreachable():
    """Over frames up to 2048 wide and targets that give a vertical box of 8 with every horizontal box 1 .. 9, uniform
    and forced, no plan names v2 at box 8 (see V2_UNREACHABLE); such plans run v4 or v1"""
    seen = set()
    for w in range(64, 2049, 92):
        for h in (w, 2 * w + 4, 16 * 9 + 7, 16 * 13 + 3):
            for f in (0.0, 0.4, 0.9):
                th = int(h / (16 + f))
                if th < 1:
                    continue
                for hs in range(1, 10):
                    tw = int(w / (2 * hs + f)) if hs > 1 else int(w / (1.2 + f))
                    if tw < 1:
                        continue
                    for geom in ((w, h, tw, th, "force"), (w, h, th * w // h or 1, None, "both")):
                        name = kernel_name(geom, True)
                        assert not name.startswith("thumbnail_fused_tma_kernel<VS=8,"), (geom, name)
                        m = re.match(r"thumbnail_fused_(mma_|tma_)?kernel<VS=8[,(]", name)
                        if m:
                            seen.add(m[1] or "")
    assert seen == {"mma_", ""}, seen


def test_wide_frames_cross_band_seams():
    """A wide frame has at least three bands and a shorter last one: v4's bands are at most 256 columns wide (the
    hook gives the exact bands of a square-target "both" plan), v1's and v2's at most 64.  Where v4 allows it, the last
    box is cut short on both axes, and at least one wide frame's last band loads TMA boxes past the frame's right edge."""
    past_edge = 0
    for fam, key, alpha, small, wide, name in CASES:
        if wide is None:
            continue
        ow, oh = out_size(wide)
        w, h = wide[:2]
        bands = v4_bands(wide) if fam == "v4" else None
        if bands is not None:
            b, reach = bands
            assert len(b) >= 3 and b[-1][1] - b[-1][0] < b[0][1] - b[0][0], (wide, b)
            past_edge += reach > w
        else:
            assert ow > (512 if fam == "v4" else 128), (wide, ow)
        if fam == "v4":
            vs, _, hs = key
            assert oh > 4 * 8 and h % vs != 0, wide     # rows_per_cta: 4 chunks of at most 8 rows
            assert w % hs != 0 or hs in (2, 4, 8), wide
        else:
            assert oh > 2 * 8, wide                     # 2 chunks of 8 rows (v1), 4 of 4 (v2)
    assert past_edge >= 1


# ------------------------------------------------------------------ GPU: every case against the oracle

N_CONTENT = 10


def contents(h, w, seed):
    """random; alpha 0, 1, 254, 255; constant 0, 255; impulses; horizontal and vertical ramps"""
    rng = np.random.default_rng(seed)
    out = [rng.integers(0, 256, (h, w, 4), dtype=np.uint8)]
    for a in (0, 1, 254, 255):
        f = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        f[..., 3] = a
        out.append(f)
    out += [np.zeros((h, w, 4), np.uint8), np.full((h, w, 4), 255, np.uint8)]
    imp = np.zeros((h, w, 4), np.uint8)
    imp[..., 3] = 255
    imp[5::13, 3::11, :3] = 255            # a lattice: within a box of every band seam
    imp[-1, ::3] = (255, 128, 7, 200)      # the last row and column
    imp[::3, -1] = (9, 255, 77, 100)
    imp[-1, -1] = 255
    out.append(imp)
    out.append(np.broadcast_to((np.arange(w) * 255 // max(1, w - 1)).astype(np.uint8)[None, :, None], (h, w, 4)).copy())
    out.append(np.broadcast_to((np.arange(h) * 255 // max(1, h - 1)).astype(np.uint8)[:, None, None], (h, w, 4)).copy())
    out[-2][..., 3] = out[-1][::-1, :, 3]  # the ramps carry live alpha
    assert len(out) == N_CONTENT
    return out


def with_seams(frames, geom):
    """the impulse frame gains an impulse column on each input column where v4's bands meet"""
    bands = v4_bands(geom)
    if bands is not None:
        for xa, xb, c_lo, c_hi in bands[0][1:]:
            frames[7][::2, c_lo, :3] = 255
            frames[7][1::2, max(0, c_lo - 1), :3] = 255
    return frames


def same(got, want, what):
    if not np.array_equal(got, want):
        d = np.argwhere(got != want)
        f, y, x, c = d[0]
        raise AssertionError("%s: %d bytes differ; first at frame %d row %d column %d channel %d (%d vs %d); rows %s, columns %s"
                             % (what, len(d), f, y, x, c, got[f, y, x, c], want[f, y, x, c], sorted(set(d[:, 1]))[:12],
                                sorted(set(d[:, 2]))[:12]))


def run_off_grid(plan, frames):
    """vb200_thumbnail_batch_device over a batch whose base pointer is 4 bytes off the 16-byte grid: v1 on this plan"""
    import torch
    n = len(frames)
    raw = torch.from_numpy(np.concatenate([np.zeros(4, np.uint8), frames.reshape(-1)])).cuda()
    out = torch.zeros((n, plan.out_height, plan.out_width, 4), dtype=torch.uint8, device="cuda")
    L = vb.lib()
    L.vb200_thumbnail_batch_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]
    vb.set_stream(torch.cuda.current_stream().cuda_stream)
    try:
        vb._check(L.vb200_thumbnail_batch_device(plan._p, raw.data_ptr() + 4, frames[0].nbytes, out.data_ptr(),
                                                 plan.out_frame_bytes, n))
        torch.cuda.synchronize()
    finally:
        vb.set_stream(0)
    return out.cpu().numpy()


def check_scale(vb, oracle, monkeypatch, fam, alpha, geom, want_name, n_batch, distinct):
    """One frame scale of a case: every content frame as a batch of one, then a batch of n_batch frames (distinct
    random frames past the content ones, or the content frames repeated), then v4's other modes on that batch"""
    w, h, tw, th, size = geom
    plan = vb.ThumbnailPlan(w, h, 4, tw, th, size=size, has_alpha=alpha)
    assert plan.kernel == want_name, plan.kernel
    base = with_seams(contents(h, w, w * 7919 + h), geom)
    if distinct:
        rng = np.random.default_rng(h * 31 + w)
        extra = rng.integers(0, 256, (n_batch - N_CONTENT, h, w, 4), dtype=np.uint8)
        extra[::3, :, :, 3] = 255          # opaque frames among the live ones
        frames = np.concatenate([np.stack(base), extra])
        want = np.stack([oracle.thumbnail_image(f, tw, th, size, has_alpha=alpha) for f in frames])
    else:
        idx = np.arange(n_batch) % N_CONTENT
        frames = np.stack(base)[idx]
        want = np.stack([oracle.thumbnail_image(f, tw, th, size, has_alpha=alpha) for f in base])[idx]
    monkeypatch.delenv("VB200_OPAQUE_PROBE", raising=False)
    monkeypatch.delenv("VB200_NO_TENSORMAP", raising=False)
    for i in range(N_CONTENT):
        same(plan.run_host(frames[i:i + 1]), want[i:i + 1], "%dx%d one frame, content %d" % (w, h, i))
    same(plan.run_host(frames), want, "%dx%d batch of %d" % (w, h, n_batch))
    if fam != "v4":
        return
    if alpha:
        for probe in ("2", "0"):
            monkeypatch.setenv("VB200_OPAQUE_PROBE", probe)
            same(plan.run_host(frames), want, "%dx%d batch, VB200_OPAQUE_PROBE=%s" % (w, h, probe))
        monkeypatch.delenv("VB200_OPAQUE_PROBE")
    monkeypatch.setenv("VB200_NO_TENSORMAP", "1")
    same(plan.run_host(frames[:1]), want[:1], "%dx%d one frame, VB200_NO_TENSORMAP" % (w, h))
    same(plan.run_host(frames), want, "%dx%d batch, VB200_NO_TENSORMAP" % (w, h))
    monkeypatch.delenv("VB200_NO_TENSORMAP")
    same(run_off_grid(plan, frames), want, "%dx%d batch, base 4 bytes off 16 (v1)" % (w, h))


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_instantiation_matches_oracle(vb, oracle, monkeypatch, case):
    import torch
    fam, key, alpha, small, wide, want_name = case
    # whole frames per CTA: rows_per_cta splits a frame's rows only while bands x frames < the CTAs it aims for (one
    # per SM for v4, two for v1 and v2); a small frame is one band, a wide one at least three
    ctas = torch.cuda.get_device_properties(0).multi_processor_count * (1 if fam == "v4" else 2)
    check_scale(vb, oracle, monkeypatch, fam, alpha, small, want_name, max(300, ctas), True)
    if wide is not None:
        check_scale(vb, oracle, monkeypatch, fam, alpha, wide, want_name, N_CONTENT * math.ceil(ctas / 3 / N_CONTENT), False)

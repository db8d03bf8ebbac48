"""Band layout of the tensor-pipe thumbnail kernel (thumbnail_fused_mma.cuh), on the CPU.

Each band CTA loads its stage rows as tiled-TMA boxes of a width fixed by the kernel's column layout, from its first
input column rounded down to the layout's alignment (a 128-byte line in the 768-column layout where shared memory
allows).  Through the host-only hook vb200_debug_thumbnail_bands this checks that the bands tile the output row, that
the boxes cover every band's input columns, and that a frame row loads no more columns than the frame has plus the
seams two bands both read plus each band's box padding."""
import ctypes as C

import pytest

import libvips_b200 as vb


def bands(width, height, target):
    L = C.CDLL(vb.library_path())
    cap = 64
    ow, nb, boxw, nbox = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    arrs = [(C.c_int * cap)() for _ in range(5)]
    L.vb200_debug_thumbnail_bands.argtypes = [C.c_int] * 3 + [C.POINTER(C.c_int)] * 2 + [C.POINTER(C.c_int)] * 5 + \
        [C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    rc = L.vb200_debug_thumbnail_bands(width, height, target, C.byref(ow), C.byref(nb), *arrs, cap, C.byref(boxw), C.byref(nbox))
    xa, xb, c_lo, c_hi, seam = ([a[i] for i in range(nb.value)] for a in arrs)
    return rc, dict(OW=ow.value, xa=xa, xb=xb, c_lo=c_lo, c_hi=c_hi, seam=seam, boxw=boxw.value, nbox=nbox.value)


def check_layout(width, height, target):
    rc, b = bands(width, height, target)
    assert rc == 0, (width, height, target)
    n = len(b["xa"])
    # the bands tile [0, OW) exactly, in order
    assert b["xa"][0] == 0 and b["xb"][-1] == b["OW"]
    assert all(b["xb"][i] == b["xa"][i + 1] for i in range(n - 1))
    assert all(b["xa"][i] < b["xb"][i] for i in range(n))
    # input columns inside the frame, 16-byte aligned starts (a 128-byte line with 416-pixel boxes), and every column of
    # the frame read by some band
    align = 32 if b["boxw"] == 416 else 4
    assert all(0 <= lo < hi <= width and lo % align == 0 for lo, hi in zip(b["c_lo"], b["c_hi"]))
    assert b["c_lo"][0] == 0 and b["c_hi"][-1] == width
    assert all(b["c_lo"][i + 1] <= b["c_hi"][i] for i in range(n - 1))
    assert all(b["seam"][i] == b["c_hi"][i] - b["c_lo"][i + 1] for i in range(n - 1)) and b["seam"][-1] == 0
    # boxes: at most 512 pixels (256 u64 elements), 16-byte rows, covering the widest band
    boxw, nbox = b["boxw"], b["nbox"]
    assert 0 < boxw <= 512 and boxw % 4 == 0 and nbox >= 1
    widest = max(hi - lo for lo, hi in zip(b["c_lo"], b["c_hi"]))
    assert widest <= nbox * boxw
    # columns a frame row loads: the frame, the seams loaded twice, the rounding of each band's boxes
    loaded = n * nbox * boxw
    assert loaded <= width + sum(b["seam"]) + sum(nbox * boxw - (hi - lo) for lo, hi in zip(b["c_lo"], b["c_hi"]))
    return b


def test_headline_bands():
    """4096 x 4096 -> 512, the bench's frame: six bands of 91 output columns, each loading from a 128-byte line (so up
    to 28 columns before the 768 its V warps read), two 416-pixel boxes -- 13 whole lines -- per stage row"""
    b = check_layout(4096, 4096, 512)
    assert b["xa"] == [0, 91, 182, 273, 364, 455]
    assert b["c_lo"] == [0, 704, 1408, 2144, 2880, 3616]
    assert [hi - lo for lo, hi in zip(b["c_lo"], b["c_hi"])] == [748, 772, 796, 788, 780, 480]
    assert b["seam"] == [44, 68, 60, 52, 44, 0]
    assert (b["nbox"], b["boxw"]) == (2, 416)
    # a frame row loads 4 992 columns: the frame's 4 096, the seams' 268 and the boxes' padding past c_hi
    assert len(b["xa"]) * b["nbox"] * b["boxw"] == 4992


@pytest.mark.parametrize("in_size,shrink", [(4096, 8.0), (2048, 8.0), (1024, 4.0), (1600, 8.0), (1000, 4.0), (4096, 8.7),
                                            (2000, 4.76), (3000, 5.9), (4096, 9.9), (4096, 16.0), (2160, 17.3)])
def test_bands_tensor_pipe_geometries(in_size, shrink):
    """the frame sizes and shrinks of the tensor-pipe table tests, as square RGBA frames"""
    rc, _ = bands(in_size, in_size, int(round(in_size / shrink)))
    if rc == 1:
        pytest.skip("this geometry does not run on the tensor-pipe kernel")
    check_layout(in_size, in_size, int(round(in_size / shrink)))


def test_bands_bad_arguments():
    assert bands(0, 4096, 512)[0] == -1

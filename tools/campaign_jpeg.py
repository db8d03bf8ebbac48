"""tools/campaign_jpeg.py SEED SECONDS -- random campaign of the JPEG decoder's and encoder's host twins (the per-block
code of jpeg.cu / jpeg_encode.cu compiled for the CPU) against libjpeg-turbo (Pillow's): random sizes, content (smooth,
noise, saturated blocks), qualities 1-100, samplings, progressive / optimised / restart-interval streams, every shrink.
Decode must be bit-exact; the encoder must write libjpeg-turbo's stream byte for byte.  TEST INFRASTRUCTURE, CPU only."""
import ctypes as C
import io
import os
import sys
import time

import numpy as np
from PIL import Image as PIL

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import libvips_b200 as vb  # noqa: E402


def content(rng, h, w, grey):
    kind = rng.integers(0, 4)
    if kind == 0:
        a = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    elif kind == 1:
        yy, xx = np.mgrid[0:h, 0:w]
        a = np.stack([128 + 100 * np.sin(xx / 37.0 + yy / 11.0), 128 + 90 * np.cos(xx / 5.0 - yy / 29.0), (xx * 3 + yy * 5) % 256], -1)
        a = np.clip(a + rng.normal(0, rng.random() * 30, a.shape), 0, 255).astype(np.uint8)
    elif kind == 2:
        a = (rng.integers(0, 2, ((h + 7) // 8, (w + 7) // 8, 3)) * 255).astype(np.uint8).repeat(8, 0).repeat(8, 1)[:h, :w]
    else:
        a = np.full((h, w, 3), rng.integers(0, 256), np.uint8)
        a[::3, ::5] = rng.integers(0, 256, 3)
    return np.ascontiguousarray(a[..., 0] if grey else a)


def turbo_decode(data, shrink):
    im = PIL.open(io.BytesIO(data))
    w, h = im.size
    if shrink > 1:
        im.draft(im.mode, (max(1, w // shrink), max(1, h // shrink)))
        if im.size != ((w + shrink - 1) // shrink, (h + shrink - 1) // shrink):
            return None
    a = np.asarray(im)[: h // shrink, : w // shrink]
    return a[..., None] if a.ndim == 2 else a


def main():
    seed = int(sys.argv[1]) if len(sys.argv) > 1 else 0
    budget = float(sys.argv[2]) if len(sys.argv) > 2 else 60.0
    rng = np.random.default_rng(seed)
    L = vb.lib()
    L.vb200_debug_jpeg_encode.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_size_t,
                                          C.POINTER(C.c_size_t)]
    t0 = time.time()
    dec = enc = bad = declined = 0
    while time.time() - t0 < budget and bad < 10:
        h, w = int(rng.integers(1, 140)), int(rng.integers(1, 140))
        grey = rng.random() < 0.2
        a = content(rng, h, w, grey)
        q = int(rng.integers(1, 101))
        sub = int(rng.integers(0, 3))
        kw = {}
        if rng.random() < 0.3:
            kw["progressive"] = True
        if rng.random() < 0.3:
            kw["optimize"] = True
        r = rng.random()
        if r < 0.25:
            kw["restart_marker_blocks"] = int(rng.integers(1, 9))
        elif r < 0.4:
            kw["restart_marker_rows"] = int(rng.integers(1, 4))
        b = io.BytesIO()
        if grey:
            PIL.fromarray(a).save(b, "JPEG", quality=q, **kw)
        else:
            PIL.fromarray(a).save(b, "JPEG", quality=q, subsampling=sub, **kw)
        d = b.getvalue()
        for shrink in (1, 2, 4, 8):
            if min(h, w) // shrink < 1:
                continue
            want = turbo_decode(d, shrink)
            if want is None:
                continue
            try:
                got = vb.jpeg_decode_host_twin(d, shrink)
            except vb.Error as e:
                declined += 1
                print("DECLINED", (h, w, grey, q, sub, kw, shrink), e, flush=True)
                continue
            dec += 1
            if got.shape != want.shape or not np.array_equal(got, want):
                bad += 1
                print("DECODE MISMATCH", (h, w, grey, q, sub, kw, shrink), got.shape, want.shape, flush=True)
        # the encoder: baseline or progressive, 4:2:0 or 4:4:4, standard or optimised tables, restart intervals of 0, 1, 2,
        # a few MCUs, or at least the MCU count
        cap = w * h * 8 + 3 * w * h // 16 + 8192
        opt = int(rng.random() < 0.5)
        interlace = int(rng.random() < 0.5)
        rmode = int(rng.integers(0, 5))
        mcus = ((w + 7) // 8) * ((h + 7) // 8)      # at least the MCU count of every sampling
        restart = [0, 1, 2, int(rng.integers(3, 12)), mcus + int(rng.integers(0, 3))][rmode]
        ekw = {}
        if opt:
            ekw["optimize"] = True
        if restart:
            ekw["restart_marker_blocks"] = restart
        if interlace:
            ekw["progressive"] = True
        buf = (C.c_ubyte * cap)()
        n = C.c_size_t()
        bands = 1 if grey else 3
        for mode, pil_sub in ((1, 2), (2, 0)) if not grey else ((0, None),):
            opts = vb.JpegSaveOptions(q, mode, opt, restart, interlace)
            rc = L.vb200_debug_jpeg_encode_opts(a.ctypes.data_as(C.c_void_p), w * bands, w, h, bands, C.byref(opts), buf, cap, C.byref(n))
            if rc:
                declined += 1
                L.vb200_error_clear()
                continue
            ours = bytes(buf[:n.value])
            t = io.BytesIO()
            if grey:
                PIL.fromarray(a).save(t, "JPEG", quality=q, **ekw)
            else:
                PIL.fromarray(a).save(t, "JPEG", quality=q, subsampling=pil_sub, **ekw)
            enc += 1
            if ours != t.getvalue():
                bad += 1
                print("ENCODE MISMATCH", (h, w, grey, q, mode, opt, restart, interlace), len(ours), len(t.getvalue()), flush=True)
    print("jpeg campaign: %d decodes, %d encodes, %d declined, %d mismatches" % (dec, enc, declined, bad))


if __name__ == "__main__":
    main()

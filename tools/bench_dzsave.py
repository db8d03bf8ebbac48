"""tools/bench_dzsave.py -- the Deep Zoom saver (vb200_dzsave / vb200_dzsave_png, csrc/dzsave.cu) on one large image.

    python tools/bench_dzsave.py [--sizes 16384,8192] [--steps 5] [--warmup 1] [--tiles jpeg|png] [--bands 3]
                                 [--kinds photo,synthetic] [--host-baseline]

A seeded, photo-like image of each size (--kinds synthetic: flat-coloured blocks and gradients, as map overlays and masks
are), saved from device memory and from pinned host memory, with the defaults (dz layout, 254 + 1 pixel tiles, Q 75 or
PNG compression 6) and as zoomify (256 pixel tiles).  --tiles png runs vb200_dzsave_png, and with it both per-batch device
budgets: the default (the PNG codecs' chunk budget) and 1 GiB (JPEG's), set with vb200_debug_dz_set_budget.
--host-baseline also times the CPU doing the same work for the dz layout -- the numpy pyramid (alpha-weighted for 2 and 4 bands) and zlib
level 6 over every tile's unfiltered scanlines on 8 threads -- and checks a sample of the device's tiles' IDAT payloads
against Python's zlib over the same scanlines.  Every vb200_dzsave call ends with the tile streams on
the host, so a call is timed with the host clock around it; ms is the median over --steps calls after --warmup calls of
the same shape.  The split into pyramid kernels / gather kernels / encoder calls / compaction and device-to-host copies
comes from a second set of calls with VB200_DZ_TIMING set, where the library brackets each phase with CUDA events (and
waits at each bracket, so those calls are not the ones the end-to-end figure is taken from).  Bytes the pyramid kernels
move are computed from the shapes: each launch reads one level and writes the next four.  The card name and power limit are
read in the same run.  One JSON line per (size, source, layout).
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import libvips_b200 as vb  # noqa: E402


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return {"gpu": name, "power_limit": limit}


def photo(size, torch, bands=3, kind="photo"):
    """photo: smooth structure + noise; synthetic: flat blocks and gradients.  Alpha (2 / 4 bands): a soft diagonal edge
    with transparent blocks.  Made on the device a band of rows at a time."""
    g = torch.Generator(device="cuda").manual_seed(size)
    out = torch.empty((size, size, bands), dtype=torch.uint8, device="cuda")
    xx = torch.arange(size, device="cuda", dtype=torch.float32)[None, :]
    for y0 in range(0, size, 1024):
        yy = torch.arange(y0, min(size, y0 + 1024), device="cuda", dtype=torch.float32)[:, None]
        if kind == "photo":
            base = torch.stack([128 + 100 * torch.sin(xx / 37 + yy / 91), 128 + 90 * torch.cos(xx / 53 - yy / 29), (xx * 3 + yy * 5) % 256], -1)
            base = base + 12 * torch.randn(base.shape, generator=g, device="cuda")
        else:
            cell = (torch.div(xx, 97, rounding_mode="floor") * 7 + torch.div(yy, 61, rounding_mode="floor") * 13) % 256
            base = torch.stack([cell, (xx / 64 + 0 * yy) % 256, (cell * 3 + yy / 32) % 256], -1)
        colour = base[..., :1].mean(-1, keepdim=True) if bands < 3 else base
        layers = [colour]
        if bands in (2, 4):
            alpha = ((xx + yy) * 255.0 / size - 64).clamp(0, 255) + 0 * yy
            hole = ((torch.div(xx, 300, rounding_mode="floor") + torch.div(yy, 300, rounding_mode="floor")) % 5 == 0)
            layers.append(torch.where(hole, torch.zeros_like(alpha), alpha)[..., None])
        out[y0:y0 + base.shape[0]] = torch.cat(layers, -1).clamp(0, 255).to(torch.uint8)
    return out


def host_levels(a):
    """the numpy pyramid from the top, a band of 2048 rows at a time (the images are gigabytes)"""
    import numpy as np
    out = [a]
    while out[-1].shape[0] > 1 or out[-1].shape[1] > 1:
        src = out[-1]
        h, w, bands = src.shape
        lvl = np.empty(((h + 1) // 2, (w + 1) // 2, bands), np.uint8)
        for y0 in range(0, h, 2048):
            p = src[y0:y0 + 2048].astype(np.int32)
            if p.shape[0] & 1:
                p = np.concatenate([p, p[-1:]], 0)
            if p.shape[1] & 1:
                p = np.concatenate([p, p[:, -1:]], 1)
            q = [p[0::2, 0::2], p[0::2, 1::2], p[1::2, 0::2], p[1::2, 1::2]]
            if bands in (2, 4):
                S = q[0][..., -1:] + q[1][..., -1:] + q[2][..., -1:] + q[3][..., -1:]
                num = sum(x[..., :-1] * x[..., -1:] for x in q)
                v = np.concatenate([num // np.maximum(S, 1), S >> 2], -1)
                v[np.broadcast_to(S == 0, v.shape)] = 0
            else:
                v = (q[0] + q[1] + q[2] + q[3] + 2) >> 2
            lvl[y0 // 2:y0 // 2 + v.shape[0]] = v
        out.append(lvl)
    return out


def scanlines(t):
    import numpy as np
    h = t.shape[0]
    return np.concatenate([np.zeros((h, 1), np.uint8), t.reshape(h, -1)], 1).tobytes()


def host_baseline(host, rects, threads=8):
    """the numpy pyramid, then zlib level 6 over each tile's scanlines on `threads` threads (zlib releases the GIL) -> ms"""
    import zlib
    from concurrent.futures import ThreadPoolExecutor
    t0 = time.perf_counter()
    levels = host_levels(host)
    top = len(levels) - 1

    def one(r):
        n, left, tp, w, h = r
        return len(zlib.compress(scanlines(levels[top - n][tp:tp + h, left:left + w]), 6))
    with ThreadPoolExecutor(threads) as ex:
        total = sum(ex.map(one, rects, chunksize=64))
    return (time.perf_counter() - t0) * 1e3, total, levels


def idat(png):
    import struct
    at, out = 8, b""
    while at < len(png):
        n, = struct.unpack(">I", png[at:at + 4])
        if png[at + 4:at + 8] == b"IDAT":
            out += png[at + 8:at + 8 + n]
        at += 12 + n
    return out


def pyramid_bytes(size, bands=3):
    """HBM bytes of the pyramid kernels: a launch reads a level once and writes up to four below it"""
    dims, moved = [size], 0
    while dims[-1] > 1:
        dims.append((dims[-1] + 1) // 2)
    for k in range(0, len(dims) - 1, 4):
        moved += bands * dims[k] ** 2 + sum(bands * d ** 2 for d in dims[k + 1:k + 5])
    return moved


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16384,8192")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--tiles", choices=("jpeg", "png"), default="jpeg")
    ap.add_argument("--bands", type=int, default=3)
    ap.add_argument("--kinds", default="photo")
    ap.add_argument("--host-baseline", action="store_true")
    args = ap.parse_args()
    png = args.tiles == "png"
    if not png and args.bands not in (1, 3):
        sys.exit("JPEG tiles take 1 or 3 bands")
    if not torch.cuda.is_available():
        sys.exit("bench_dzsave needs a GPU: there is no CPU path to time")
    vb.init(0)
    L = vb.lib()
    where = card()
    bands = args.bands
    pngo = vb._png_options(6, "default", 1.0)
    for size, kind in [(int(s), k) for s in args.sizes.split(",") for k in args.kinds.split(",")]:
        dev = photo(size, torch, bands, kind)
        host = dev.cpu().pin_memory()
        if args.host_baseline and png:
            import numpy as np
            a = host.numpy()
            for layout in ("dz",):
                cin = vb.CImage(size, size, bands, 0, 1 if bands < 3 else 22, vb.DEVICE, C.c_void_p(dev.data_ptr()), size * bands)
                handle = C.c_void_p()
                vb._check(L.vb200_dzsave_png(C.byref(cin), C.byref(vb.DzOptions(vb.DZ_LAYOUTS[layout], 0, -1, 0, 0, 0, 0, None)), C.byref(pngo),
                                             C.byref(handle)))
                p = vb.DzPyramid(handle, None)
                rects = [(t.level,) + t.rect for t in p.tiles]
                ms, zbytes, levels = host_baseline(a, rects)
                top = len(levels) - 1
                rng = np.random.default_rng(size)
                sample = rng.choice(len(p.tiles), min(64, len(p.tiles)), replace=False)
                ok = all(idat(p.tiles[i].bytes) == zlib.compress(scanlines(levels[top - r[0]][r[2]:r[2] + r[4], r[1]:r[1] + r[3]]), 6)
                         for i, r in ((i, rects[i]) for i in sample))
                print(json.dumps(dict(where, size=size, kind=kind, bands=bands, layout=layout, source="host baseline", tiles=len(rects),
                                      ms=round(ms, 1), tiles_per_s=round(len(rects) / ms * 1e3), threads=8, zlib_bytes=zbytes,
                                      device_bytes=sum(len(t.bytes) for t in p.tiles), sample_tiles_equal_python_zlib=bool(ok),
                                      sample=len(sample))), flush=True)
                del p, levels
        for source, ptr, loc in (("device", dev.data_ptr(), vb.DEVICE), ("pinned host", host.data_ptr(), vb.HOST)):
            for layout, budget in [(l, b) for l in ("dz", "zoomify") for b in ((0, 1 << 30) if png else (0,))]:
                cin = vb.CImage(size, size, bands, 0, 1 if bands < 3 else 22, loc, C.c_void_p(ptr), size * bands)
                opts = vb.DzOptions(vb.DZ_LAYOUTS[layout], 0, -1, 0, 0, 0, 0, None, vb.JpegSaveOptions(75, 0, 0, 0, 0))
                L.vb200_debug_dz_set_budget(budget)

                def call():
                    handle = C.c_void_p()
                    t0 = time.perf_counter()
                    if png:
                        vb._check(L.vb200_dzsave_png(C.byref(cin), C.byref(opts), C.byref(pngo), C.byref(handle)))
                    else:
                        vb._check(L.vb200_dzsave(C.byref(cin), C.byref(opts), C.byref(handle)))
                    ms = (time.perf_counter() - t0) * 1e3
                    tiles = L.vb200_dz_tiles(handle)
                    L.vb200_dz_free(handle)
                    return ms, tiles
                os.environ.pop("VB200_DZ_TIMING", None)
                for _ in range(args.warmup):
                    call()
                before = vb.launch_count()
                runs = [call() for _ in range(args.steps)]
                launches = (vb.launch_count() - before) // args.steps
                ms, tiles = statistics.median(r[0] for r in runs), runs[0][1]
                os.environ["VB200_DZ_TIMING"] = "1"
                split = []
                for _ in range(max(1, args.steps // 2)):
                    call()
                    t = (C.c_float * 4)()
                    L.vb200_debug_dz_times(t)
                    split.append(list(t))
                os.environ.pop("VB200_DZ_TIMING", None)
                phase = [statistics.median(s[k] for s in split) for k in range(4)]
                L.vb200_debug_dz_set_budget(0)
                print(json.dumps(dict(where, size=size, kind=kind, bands=bands, tiles_format=args.tiles, budget="default" if budget == 0 else budget,
                                      source=source, layout=layout, tiles=tiles, ms=round(ms, 2), ms_min=round(min(r[0] for r in runs), 2),
                                      ms_max=round(max(r[0] for r in runs), 2), tiles_per_s=round(tiles / ms * 1e3),
                                      input_mpixels_per_s=round(size * size / ms / 1e3), launches=launches,
                                      pyramid_ms=round(phase[0], 3), gather_ms=round(phase[1], 3), encode_ms=round(phase[2], 3),
                                      d2h_ms=round(phase[3], 3),
                                      pyramid_gb_per_s=round(pyramid_bytes(size, bands) / phase[0] / 1e6, 1) if phase[0] > 0 else None,
                                      steps=args.steps, warmup=args.warmup)), flush=True)
        del dev, host
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

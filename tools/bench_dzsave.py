"""tools/bench_dzsave.py -- the Deep Zoom saver (vb200_dzsave, csrc/dzsave.cu) on one large image.

    python tools/bench_dzsave.py [--sizes 16384,8192] [--steps 5] [--warmup 1]

A seeded, photo-like RGB image of each size, saved from device memory and from pinned host memory, with the defaults (dz
layout, 254 + 1 pixel tiles, Q 75) and as zoomify (256 pixel tiles).  Every vb200_dzsave call ends with the tile streams on
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


def photo(size, torch):
    """smooth structure + noise, made on the device a band of rows at a time"""
    g = torch.Generator(device="cuda").manual_seed(size)
    out = torch.empty((size, size, 3), dtype=torch.uint8, device="cuda")
    xx = torch.arange(size, device="cuda", dtype=torch.float32)[None, :]
    for y0 in range(0, size, 1024):
        yy = torch.arange(y0, min(size, y0 + 1024), device="cuda", dtype=torch.float32)[:, None]
        base = torch.stack([128 + 100 * torch.sin(xx / 37 + yy / 91), 128 + 90 * torch.cos(xx / 53 - yy / 29), (xx * 3 + yy * 5) % 256], -1)
        base = base + 12 * torch.randn(base.shape, generator=g, device="cuda")
        out[y0:y0 + base.shape[0]] = base.clamp(0, 255).to(torch.uint8)
    return out


def pyramid_bytes(size):
    """HBM bytes of the pyramid kernels: a launch reads a level once and writes up to four below it"""
    dims, moved = [size], 0
    while dims[-1] > 1:
        dims.append((dims[-1] + 1) // 2)
    for k in range(0, len(dims) - 1, 4):
        moved += 3 * dims[k] ** 2 + sum(3 * d ** 2 for d in dims[k + 1:k + 5])
    return moved


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16384,8192")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_dzsave needs a GPU: there is no CPU path to time")
    vb.init(0)
    L = vb.lib()
    where = card()
    for size in [int(s) for s in args.sizes.split(",")]:
        dev = photo(size, torch)
        host = dev.cpu().pin_memory()
        for source, ptr, loc in (("device", dev.data_ptr(), vb.DEVICE), ("pinned host", host.data_ptr(), vb.HOST)):
            for layout in ("dz", "zoomify"):
                cin = vb.CImage(size, size, 3, 0, 22, loc, C.c_void_p(ptr), size * 3)
                opts = vb.DzOptions(vb.DZ_LAYOUTS[layout], 0, -1, 0, 0, 0, 0, None, vb.JpegSaveOptions(75, 0, 0, 0, 0))

                def call():
                    handle = C.c_void_p()
                    t0 = time.perf_counter()
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
                print(json.dumps(dict(where, size=size, source=source, layout=layout, tiles=tiles, ms=round(ms, 2), ms_min=round(min(r[0] for r in runs), 2),
                                      ms_max=round(max(r[0] for r in runs), 2), tiles_per_s=round(tiles / ms * 1e3),
                                      input_mpixels_per_s=round(size * size / ms / 1e3), launches=launches,
                                      pyramid_ms=round(phase[0], 3), gather_ms=round(phase[1], 3), encode_ms=round(phase[2], 3),
                                      d2h_ms=round(phase[3], 3), pyramid_gb_per_s=round(pyramid_bytes(size) / phase[0] / 1e6, 1) if phase[0] > 0 else None,
                                      steps=args.steps, warmup=args.warmup)), flush=True)
        del dev, host
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

"""tools/bench_hist.py -- the histogram ops on the device (csrc/histogram.cu) against the reference's own sources on the
host.

    python tools/bench_hist.py [--reps R] [--threads T] [--out DIR]

Workloads, every input device-resident and every output left on the device (library-allocated):
    hist_local  4096 x 4096 RGB uchar, 64 x 64 window, max_slope 3 (sharp's clahe() default)
    hist_equal  4096 x 4096 RGB uchar, and 4096 x 4096 one-band ushort
    hist_find   4096 x 4096 RGB uchar, and 4096 x 4096 one-band ushort
Device frames/s come from CUDA events around R calls after a warm-up call.  The host side runs the reference's own
hist_local.c under oracle/_ref (where it has been built) on T threads, each on a band of rows with its window's halo:
hist_local's rows are independent, so the bands' interiors are the whole image's rows.  The card's name and power limit
are read in the same run.  One JSON line per workload; with --out, a summary in DIR/bench_hist.json."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = __file__.rsplit("/tools/", 1)[0]
sys.path.insert(0, ROOT)
import libvips_b200 as vb  # noqa: E402


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the card's name still says what ran
        q = "unknown (%s)" % e
    return name, q


def photo(h, w, bands, dt, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    base = np.stack([128 + 100 * np.sin(x / (37 + 13 * c) + y / (53 + 7 * c) + c) for c in range(bands)], 2)
    a = np.clip(base + rng.normal(0, 6, base.shape), 0, 255)
    return (a * (257 if dt == np.uint16 else 1)).astype(dt)


def device_fps(a, call, reps):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).cuda()
    h, w, b = a.shape
    cin = vb.CImage(w, h, b, vb.FORMATS[a.dtype], 22 if b == 3 else 1, vb.DEVICE, C.c_void_p(t.data_ptr()), w * b * a.itemsize)
    vb.set_stream(torch.cuda.current_stream().cuda_stream)

    def once():
        cout = vb.CImage()
        cout.where = vb.DEVICE
        vb._check(call(C.byref(cin), C.byref(cout)))
        vb.lib().vb200_image_free(C.byref(cout))

    once()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        once()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    return 1000.0 / ms, ms


def host_hist_local_fps(a, ww, wh, m, threads, reps):
    """the reference's hist_local.c on `threads` row bands with halo (None where oracle/_ref is not built)"""
    path = os.path.join(ROOT, "oracle", "_ref", "libvipsref.so")
    if not os.path.exists(path):
        return None
    L = C.CDLL(path)
    L.ref_image_new_from_memory.restype = C.c_void_p
    L.ref_image_new_from_memory.argtypes = [C.c_void_p] + [C.c_int] * 5
    L.ref_hist_local.restype = C.c_void_p
    L.ref_hist_local.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.ref_image_write_to_memory.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    h, w, b = a.shape
    out = np.empty_like(a)
    step = (h + threads - 1) // threads

    def band(y0):
        y1 = min(h, y0 + step)
        s0, s1 = max(0, y0 - wh // 2), min(h, y1 + wh - wh // 2 - 1)
        sl = np.ascontiguousarray(a[s0:s1])
        im = L.ref_image_new_from_memory(sl.ctypes.data, w, s1 - s0, b, 0, 22)
        o = L.ref_hist_local(im, ww, wh, m)
        res = np.empty_like(sl)
        L.ref_image_write_to_memory(o, res.ctypes.data, 0, 0)
        out[y0:y1] = res[y0 - s0:y0 - s0 + (y1 - y0)]

    def once():
        with ThreadPoolExecutor(threads) as ex:
            list(ex.map(band, range(0, h, step)))

    once()
    t0 = time.perf_counter()
    for _ in range(reps):
        once()
    return reps / (time.perf_counter() - t0), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--threads", type=int, default=8)
    ap.add_argument("--host-reps", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    vb.init(0)
    name, power = card()
    L = vb.lib()
    rgb = photo(4096, 4096, 3, np.uint8, 1)
    grey16 = photo(4096, 4096, 1, np.uint16, 2)
    rows = []
    work = [("hist_local 4096x4096 RGB 64x64 max_slope 3", rgb, lambda i, o: L.vb200_hist_local(i, o, 64, 64, 3)),
            ("hist_equal 4096x4096 RGB uchar", rgb, lambda i, o: L.vb200_hist_equal(i, o, -1)),
            ("hist_equal 4096x4096 ushort", grey16, lambda i, o: L.vb200_hist_equal(i, o, -1)),
            ("hist_find 4096x4096 RGB uchar", rgb, lambda i, o: L.vb200_hist_find(i, o, -1)),
            ("hist_find 4096x4096 ushort", grey16, lambda i, o: L.vb200_hist_find(i, o, -1))]
    for what, a, call in work:
        fps, ms = device_fps(a, call, args.reps)
        row = {"workload": what, "device_fps": round(fps, 2), "device_ms": round(ms, 3), "gpu": name, "power_limit": power}
        if what.startswith("hist_local"):
            host = host_hist_local_fps(a, 64, 64, 3, args.threads, args.host_reps)
            if host is not None:
                row["host_ref_fps"] = round(host[0], 3)
                row["host_threads"] = args.threads
                row["device_equals_host_ref"] = bool(np.array_equal(vb.Image(a).hist_local(64, 64, 3).numpy(), host[1]))
            else:
                row["host_ref_fps"] = "not measured (oracle/_ref not built)"
        print(json.dumps(row), flush=True)
        rows.append(row)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_hist.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()

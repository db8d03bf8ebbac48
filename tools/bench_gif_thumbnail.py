"""tools/bench_gif_thumbnail.py -- animated GIF thumbnails (every page, n = -1) on the device against libnsgif plus the
reference chain's resize on the host's own threads.

    python tools/bench_gif_thumbnail.py [--reps R] [--threads T] [--out DIR]

Workloads (animations written by Pillow from a seed; a few distinct streams repeated to fill a batch):
    small   1024 GIFs of 16 frames at 320 x 240, to width 128
    long    64 GIFs of 100 frames at 480 x 270, to width 200
Device: ThumbnailPlan(page_height = screen height).run_gif(streams, n = -1) into device memory -- LZW, composition and the
page-strip thumbnail without the frames leaving the device.  Host: each stream decoded by libnsgif through the oracle built
under oracle/_ref (the strip nsgifload gives with n = -1), then premultiply / resize / unpremultiply of the whole strip by the
oracle port (liboracle_fast.so, -O3 -march=native) with the same page-height shrinks, one stream per thread as bench.py's
cpu_baseline runs frames.  Reports animated thumbnails/s and pages/s for both; the card's name and power limit are read in
the same run.  One JSON line per workload; with --out, a summary in DIR/bench_gif_thumbnail.json."""
import argparse
import ctypes as C
import io
import json
import os
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
from PIL import Image as PIL

ROOT = __file__.rsplit("/tools/", 1)[0]
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import libvips_b200 as vb  # noqa: E402
from bench_gifload import card, host_timed, nsgif_lib, timed  # noqa: E402


def animation(W, H, frames, seed):
    """a moving pattern over a noisy field, drawn straight in one 256-colour palette"""
    rng = np.random.default_rng(seed)
    pal = rng.integers(0, 256, 768, dtype=np.uint8).tobytes()
    y, x = np.mgrid[0:H, 0:W].astype(np.float32)
    ims = []
    for k in range(frames):
        field = 128 + 100 * np.sin((x + 3 * k) / (37 + seed) + (y - 2 * k) / 53) + rng.normal(0, 8, (H, W))
        im = PIL.fromarray(np.clip(field, 0, 255).astype(np.uint8), "P")
        im.putpalette(pal)
        ims.append(im)
    b = io.BytesIO()
    ims[0].save(b, "GIF", save_all=True, append_images=ims[1:], duration=40, loop=0, disposal=1, optimize=False)
    return b.getvalue()


def oracle_fast():
    from oracle import pyoracle
    path = os.path.join(ROOT, "oracle", "liboracle_fast.so")
    if not os.path.exists(path):
        pyoracle.build()
    return C.CDLL(path)


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    vb.init(0)
    name, limit = card()
    ns = nsgif_lib()
    F = oracle_fast()
    results = []
    for label, n, W, H, frames, target in (("small", 1024, 320, 240, 16, 128), ("long", 64, 480, 270, 100, 200)):
        distinct = [animation(W, H, frames, i) for i in range(8)]
        geo = vb.gif_geometry(distinct[0])
        distinct = [s for s in distinct if vb.gif_geometry(s) == geo]
        streams = [distinct[i % len(distinct)] for i in range(n)]
        batch = vb.StreamBatch(streams)
        w, h, bands, fc = geo
        plan = vb.ThumbnailPlan(w, h * fc, bands, target, page_height=h)
        ow, oh = plan.out_width, plan.out_height
        dev = torch.empty(n * plan.out_frame_bytes, dtype=torch.uint8, device="cuda")
        t_dev = timed(lambda: plan.run_gif(batch, out_ptr=dev.data_ptr(), n=-1), args.reps)
        got = dev.view(n, oh, ow, plan.out_bands)[n - 1].cpu().numpy()

        # the host chain: libnsgif's strip, then the oracle port's page-strip thumbnail
        hs, vs, _, _, _ = vb.thumbnail_pages_size(w, h, fc, target)
        premul = bands == 4 and hs != 1.0 and vs != 1.0

        def host_one(s):
            strip = np.empty((h * fc, w, bands), np.uint8)
            info = (C.c_int * 5)()
            if ns.nsgif_oracle_load(s, len(s), 0, -1, strip.ctypes.data, info, None, 0):
                raise RuntimeError("libnsgif failed")
            src = strip
            if premul:
                src = np.empty_like(strip)
                F.orc_premultiply(C.c_void_p(strip.ctypes.data), w, h * fc, bands, 0, C.c_double(255.0), 1, C.c_void_p(src.ctypes.data))
            out = np.empty((oh, ow, bands), np.uint8)
            rc = F.orc_resize(C.c_void_p(src.ctypes.data), w, h * fc, bands, 0, C.c_double(1.0 / hs), C.c_double(1.0 / vs), 5,
                              C.c_double(2.0), 0, 0, C.c_void_p(out.ctypes.data))
            if rc:
                raise RuntimeError("oracle resize failed")
            if premul:
                res = out
                out = np.empty_like(res)
                F.orc_unpremultiply(C.c_void_p(res.ctypes.data), ow, oh, bands, 0, C.c_double(255.0), 1, C.c_void_p(out.ctypes.data))
            return out

        t_host = None
        if ns is not None:
            assert np.array_equal(got, host_one(streams[n - 1])), "device thumbnail differs from the host chain"
            pool = ThreadPoolExecutor(args.threads)
            t_host = host_timed(lambda: list(pool.map(host_one, streams)), 1)
            pool.shutdown()
        plan.close()
        r = {"workload": "%s_%dx%d_%dframes_to_%d" % (label, W, H, frames, target), "streams": n, "pages_per_stream": fc, "bands": bands,
             "kernel": plan.kernel, "out": [oh, ow], "out_page_height": plan.out_page_height,
             "compressed_MB": round(batch.nbytes / 1e6, 2),
             "device_thumbnails_per_s": round(n / t_dev[0], 1), "device_pages_per_s": round(n * fc / t_dev[0], 1),
             "device_s": [round(v, 4) for v in t_dev],
             "host_thumbnails_per_s": round(n / t_host, 1) if t_host else "not measured (oracle/_ref not built)",
             "host_pages_per_s": round(n * fc / t_host, 1) if t_host else "not measured (oracle/_ref not built)",
             "host_threads": args.threads, "gpu": name, "power_limit_max_sm_clock": limit}
        print(json.dumps(r), flush=True)
        results.append(r)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_gif_thumbnail.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()

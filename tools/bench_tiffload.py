"""tools/bench_tiffload.py -- TIFF decode on the device (csrc/tiff.cu) against Pillow's libtiff on 8 host threads.

    python tools/bench_tiffload.py [--reps R] [--slide N] [--out DIR]

Workloads (streams from tests/test_tiff.py's writer, a few distinct ones repeated to fill a batch):
    small   batches of 2 048 256 x 256 RGB TIFFs in 64 x 64 tiles: deflate + predictor 2, LZW, and JPEG (4:2:0, JPEGTables)
    slide   one N x N (default 16384) RGB TIFF in 256 x 256 deflate tiles: decode time, and as a subifd and a page pyramid,
            vb.thumbnail_buffer to 256 pixels in thumbnails/s; the same slide in 256 x 256 JPEG tiles: decode time and its
            subifd pyramid's thumbnail
The card's name and power limit are read in the same run.  One JSON line per workload; with --out, a summary in DIR/bench_tiffload.json."""
import argparse
import io
import json
import os
import subprocess
import sys
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np
from PIL import Image as PIL

ROOT = __file__.rsplit("/tools/", 1)[0]
sys.path.insert(0, ROOT)
sys.path.insert(0, ROOT + "/tests")
import libvips_b200 as vb  # noqa: E402
import test_tiff as T  # noqa: E402


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the card's name still says what ran
        q = "unknown (%s)" % e
    return name, q


def photo(h, w, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    base = np.stack([128 + 100 * np.sin(x / (37 + 13 * c) + y / (53 + 7 * c) + c) for c in range(3)], 2)
    return np.clip(base + rng.normal(0, 6, base.shape), 0, 255).astype(np.uint8)


def timed(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    best = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best.append(time.perf_counter() - t0)
    return float(np.median(best))


def pillow_decode(streams, threads=8):
    def one(s):
        return np.asarray(PIL.open(io.BytesIO(s)).convert("RGB"))
    with ThreadPoolExecutor(threads) as ex:
        list(ex.map(one, streams))


def jpeg_tiff(a, tile, subifds=(), big=False):
    """a tiled YCbCr JPEG TIFF at quality 85, 4:2:0, with JPEGTables; subifds: further levels as tiled JPEG SubIFDs"""
    def page(x):
        segs, tab, _ = T.jpeg_tiles(x, (tile, tile), 2, True)
        return T.Page(x, 6, comp=7, tile=(tile, tile), segments=segs, tags={347: (7, list(tab))})
    top = page(a)
    top.subifds = [page(x) for x in subifds]
    return T.make_tiff([top], "<", big)


def small(reps, results):
    import torch
    for name, comp, pred in (("deflate+pred", 8, 2), ("lzw", 5, 1), ("jpeg", 7, 1)):
        distinct = [T.make_tiff([T.Page(photo(256, 256, i), comp=comp, pred=pred, tile=(64, 64))]) if comp != 7 else jpeg_tiff(photo(256, 256, i), 64)
                    for i in range(8)]
        streams = [distinct[i % 8] for i in range(2048)]
        batch = vb.StreamBatch(streams)
        dev = torch.empty(2048 * 256 * 256 * 3, dtype=torch.uint8, device="cuda")
        t = timed(lambda: vb.tiff_decode_batch(batch, out_ptr=dev.data_ptr()), reps)
        t0 = time.perf_counter()
        pillow_decode(streams)
        th = time.perf_counter() - t0
        r = {"workload": "small-" + name, "frames": 2048, "device_frames_per_s": 2048 / t, "host_pillow_8t_frames_per_s": 2048 / th,
             "mean_stream_bytes": batch.nbytes / 2048}
        print(json.dumps(r), flush=True)
        results.append(r)


def slide(n, reps, results):
    import torch
    a = photo(n, n, 7)
    tile = 256

    def tiles(img):
        h, w, _ = img.shape
        segs = []
        for y in range(0, h, tile):
            for x in range(0, w, tile):
                t = np.zeros((tile, tile, 3), np.uint8)
                p = img[y:y + tile, x:x + tile]
                t[:p.shape[0], :p.shape[1]] = p
                segs.append(t)
        with ThreadPoolExecutor(os.cpu_count() or 8) as ex:
            return list(ex.map(lambda t: zlib.compress(T.difference(t).tobytes(), 1), segs))

    levels = [a]
    while levels[-1].shape[0] > 256:
        levels.append(np.ascontiguousarray(levels[-1][::2, ::2]))
    pages = [T.Page(l, comp=8, pred=2, tile=(tile, tile), segments=tiles(l)) for l in levels]
    flat = T.make_tiff([pages[0]], "<", True)
    sub = T.make_tiff([T.Page(levels[0], comp=8, pred=2, tile=(tile, tile), segments=pages[0].segments, subifds=pages[1:])], "<", True)
    pyr = T.make_tiff(pages, "<", True)
    dev = torch.empty(n * n * 3, dtype=torch.uint8, device="cuda")
    t = timed(lambda: vb.tiff_decode_batch([flat], out_ptr=dev.data_ptr()), reps)
    t0 = time.perf_counter()
    PIL.MAX_IMAGE_PIXELS = None
    try:
        np.asarray(PIL.open(io.BytesIO(flat)).convert("RGB"))
        th = time.perf_counter() - t0
    except Exception as e:  # Pillow may refuse a file this size
        th = None
        print("pillow: %s" % e, file=sys.stderr)
    r = {"workload": "slide-%d-deflate" % n, "device_decode_s": t, "host_pillow_decode_s": th, "stream_bytes": len(flat)}
    print(json.dumps(r), flush=True)
    results.append(r)
    jflat = jpeg_tiff(a, tile, big=True)
    jsub = jpeg_tiff(a, tile, levels[1:], big=True)
    t = timed(lambda: vb.tiff_decode_batch([jflat], out_ptr=dev.data_ptr()), reps)
    t0 = time.perf_counter()
    try:
        np.asarray(PIL.open(io.BytesIO(jflat)).convert("RGB"))
        th = time.perf_counter() - t0
    except Exception as e:  # Pillow may refuse a file this size
        th = None
        print("pillow: %s" % e, file=sys.stderr)
    r = {"workload": "slide-%d-jpeg" % n, "device_decode_s": t, "host_pillow_decode_s": th, "stream_bytes": len(jflat)}
    print(json.dumps(r), flush=True)
    results.append(r)
    for name, s in (("subifd", sub), ("page", pyr), ("flat", flat), ("jpeg-subifd", jsub)):
        level = vb.thumbnail_tiff_level(s, 256)
        tt = timed(lambda: vb.thumbnail_buffer(s, 256), reps)
        r = {"workload": "slide-%d-thumbnail-%s" % (n, name), "level": level, "thumbnails_per_s": 1 / tt}
        print(json.dumps(r), flush=True)
        results.append(r)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--slide", type=int, default=16384)
    ap.add_argument("--out")
    args = ap.parse_args()
    vb.init(0)
    name, power = card()
    print(json.dumps({"card": name, "power_limit": power}), flush=True)
    results = []
    small(args.reps, results)
    slide(args.slide, args.reps, results)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_tiffload.json"), "w") as f:
            json.dump({"card": name, "power_limit": power, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()

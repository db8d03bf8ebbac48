"""tools/bench_webpload.py -- WebP decode on the device (csrc/webp.cu) against Pillow's libwebp on 8 host threads.

    python tools/bench_webpload.py [--reps R] [--kernels] [--out DIR]

Workloads (Pillow-encoded lossy streams, one token partition each, a few distinct ones repeated to fill a batch):
    small   a batch of 2 048 256 x 256 frames at quality 75 and at quality 95
    large   a batch of 16 4096 x 4096 frames at quality 75 and at quality 95
Device frames/s are with the output left on the device; both sides are warmed up once and timed as the median of --reps
runs, the host on one pool of 8 threads.  With --kernels, each workload's device time is also split per kernel
(the library's CUDA events, VB200_WEBP_TIMING, over one batch).  The card's name and power limit are read in the same run.  One JSON line per workload;
with --out, a summary in DIR/bench_webpload.json."""
import argparse
import io
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
from PIL import Image as PIL

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


def photo(h, w, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    base = np.stack([128 + 100 * np.sin(x / (37 + 13 * c) + y / (53 + 7 * c) + c) for c in range(3)], 2)
    return np.clip(base + rng.normal(0, 6, base.shape), 0, 255).astype(np.uint8)


def webp(a, q):
    b = io.BytesIO()
    PIL.fromarray(a).save(b, "WEBP", quality=q)
    return b.getvalue()


def timed(fn, reps, sync):
    fn()
    sync()
    best = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        sync()
        best.append(time.perf_counter() - t0)
    return float(np.median(best))


def one(s):
    return np.asarray(PIL.open(io.BytesIO(s)).convert("RGB"))


def kernel_split(fn):
    """device milliseconds per kernel over one call of fn (the library's CUDA events, VB200_WEBP_TIMING)"""
    os.environ["VB200_WEBP_TIMING"] = "1"
    try:
        fn()
        return vb.webp_times()
    finally:
        del os.environ["VB200_WEBP_TIMING"]


def run(name, side, n, distinct, q, reps, results, pool, kernels):
    import torch
    d = [webp(photo(side, side, i), q) for i in range(distinct)]
    streams = [d[i % distinct] for i in range(n)]
    batch = vb.StreamBatch(streams)
    dev = torch.empty(n * side * side * 3, dtype=torch.uint8, device="cuda")
    decode = lambda: vb.webp_decode_batch(batch, out_ptr=dev.data_ptr())  # noqa: E731
    t = timed(decode, reps, torch.cuda.synchronize)
    th = timed(lambda: list(pool.map(one, streams)), reps, lambda: None)
    r = {"workload": "%s-q%d" % (name, q), "frames": n, "side": side, "device_frames_per_s": n / t, "host_pillow_8t_frames_per_s": n / th,
         "mean_stream_bytes": batch.nbytes / n}
    if kernels:
        r["kernel_ms_per_batch"] = kernel_split(decode)
    print(json.dumps(r), flush=True)
    results.append(r)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--kernels", action="store_true", help="split each workload's device time per kernel")
    args = ap.parse_args()
    vb.init(0)
    name, power = card()
    print(json.dumps({"card": name, "power_limit": power}), flush=True)
    results = []
    with ThreadPoolExecutor(8) as pool:
        for q in (75, 95):
            run("small", 256, 2048, 8, q, args.reps, results, pool, args.kernels)
            run("large", 4096, 16, 2, q, args.reps, results, pool, args.kernels)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_webpload.json"), "w") as f:
            json.dump({"card": name, "power_limit": power, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()

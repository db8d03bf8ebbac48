"""tools/bench_pngload.py -- PNG decode on the device (csrc/png.cu) against Pillow's decoder on the host's own threads.

    python tools/bench_pngload.py [--reps R] [--out DIR]

Workloads (PNGs written by Pillow at compress_level 6 from a seed; a few distinct streams repeated to fill a batch):
    big     4096 x 4096 RGBA and RGB, synthetic (smooth gradients and flat runs) and photo-like (noise over smooth fields)
    small   256 x 256 RGBA and RGB, the same two contents
Reports, per workload: device decode frames/s and decoded GB/s (vb.png_decode_batch into device memory), Pillow's
decode of the same streams on the machine's threads, ThumbnailPlan.run_png end to end (to 128 pixels), and the split
between the inflate and unfilter / expand kernels from a separate torch.profiler pass.  The card's name and power limit are
read in the same run.  One JSON line per workload; with --out, a summary in DIR/bench_pngload.json."""
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

sys.path.insert(0, __file__.rsplit("/tools/", 1)[0])
import libvips_b200 as vb  # noqa: E402


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the card's name still says what ran
        q = "unknown (%s)" % e
    return name, q


def content(kind, h, w, bands, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    if kind == "synthetic":
        a = np.stack([(x * 255 / w), (y * 255 / h), ((x + y) * 127 / (w + h)), 255 - x * 200 / w], 2)[:, :, :bands]
        a[h // 3:h // 2, :, :] = 40  # a flat run
        return a.astype(np.uint8)
    base = np.stack([128 + 100 * np.sin(x / (37 + 13 * c) + y / (53 + 7 * c) + c) for c in range(bands)], 2)
    return np.clip(base + rng.normal(0, 12, base.shape), 0, 255).astype(np.uint8)


def streams_of(kind, size, bands, distinct):
    out = []
    for i in range(distinct):
        b = io.BytesIO()
        PIL.fromarray(content(kind, size, size, bands, i), "RGBA" if bands == 4 else "RGB").save(b, "PNG", compress_level=6)
        out.append(b.getvalue())
    return out


def timed(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        t.append(time.perf_counter() - t0)
    return float(np.median(t)), float(min(t)), float(max(t))


def kernel_split(batch, dev):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        vb.png_decode_batch(batch, out_ptr=dev.data_ptr())
        torch.cuda.synchronize()
    ms = {}
    for e in prof.key_averages():
        for k in ("png_inflate_kernel", "png_unfilter_kernel", "png_expand_kernel"):
            if k in e.key:
                ms[k] = ms.get(k, 0.0) + getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1000.0
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None, help="directory for bench_pngload.json (default: print only)")
    ap.add_argument("--big-frames", type=int, default=16)
    ap.add_argument("--small-frames", type=int, default=2048)
    args = ap.parse_args()
    import torch
    vb.init(0)
    name, limit = card()
    threads = len(os.sched_getaffinity(0))
    print(json.dumps({"card": name, "power_limit_and_max_sm_clock": limit, "host_threads": threads}), flush=True)
    results = []
    for size, n in ((256, args.small_frames), (4096, args.big_frames)):
        for bands in (4, 3):
            for kind in ("synthetic", "photo"):
                distinct = 8 if size <= 256 else 2
                ss = streams_of(kind, size, bands, distinct)
                batch = vb.StreamBatch([ss[i % distinct] for i in range(n)])
                frame = size * size * bands
                dev = torch.empty(frame * n, dtype=torch.uint8, device="cuda")
                med, lo, hi = timed(lambda: vb.png_decode_batch(batch, out_ptr=dev.data_ptr()), args.reps)
                ok = bool(np.array_equal(dev[:frame].cpu().numpy().reshape(size, size, bands), np.array(PIL.open(io.BytesIO(ss[0])))))
                split = kernel_split(batch, dev)

                def pillow_all():
                    with ThreadPoolExecutor(threads) as ex:
                        list(ex.map(lambda s: np.asarray(PIL.open(io.BytesIO(s)).convert("RGBA" if bands == 4 else "RGB")), batch.streams))
                t0 = time.perf_counter()
                pillow_all()
                host_s = time.perf_counter() - t0
                plan = vb.ThumbnailPlan(size, size, bands, 128)
                out = torch.empty(plan.out_frame_bytes * n, dtype=torch.uint8, device="cuda")
                th_med, _, _ = timed(lambda: plan.run_png(batch, out_ptr=out.data_ptr()), 1)
                plan.close()
                del dev, out
                r = {"workload": "%s %dx%d %s" % (kind, size, size, "RGBA" if bands == 4 else "RGB"), "frames": n,
                     "compressed_MB_per_frame": round(batch.nbytes / n / 1e6, 3), "device_s": round(med, 4), "device_s_min_max": [round(lo, 4), round(hi, 4)],
                     "device_frames_per_s": round(n / med, 1), "device_decoded_GB_per_s": round(frame * n / med / 1e9, 3),
                     "kernel_ms": {k: round(v, 2) for k, v in split.items()}, "pillow_threads": threads, "pillow_s": round(host_s, 4),
                     "pillow_frames_per_s": round(n / host_s, 1), "run_png_128_s": round(th_med, 4), "run_png_frames_per_s": round(n / th_med, 1),
                     "first_frame_equals_pillow": ok}
                print(json.dumps(r), flush=True)
                results.append(r)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_pngload.json"), "w") as f:
            json.dump({"card": name, "power_limit_and_max_sm_clock": limit, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()

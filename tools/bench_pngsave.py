"""tools/bench_pngsave.py -- PNG save on the device (csrc/png_encode.cu) against zlib on the host's own threads.

    python tools/bench_pngsave.py [--reps R] [--out DIR] [--small N] [--big N] [--filter F] [--interlace]

Workloads (frames from a seed, compression 6, Z_DEFAULT_STRATEGY; filter NONE and not interlaced unless --filter sub / up /
avg / paeth or --interlace say otherwise, which then apply to every workload):
    small   N (2048) 256 x 256 RGBA and RGB frames in device memory, synthetic (smooth gradients and flat runs) and
            photo-like (noise over smooth fields)
    big     N (16) 4096 x 4096 RGB frames, the same two contents
    e2e     PNG streams -> ThumbnailPlan.run_png (to 256 pixels) -> pngsave_batch: streams in, streams out
The baseline is zlib level 6 over the same scanlines on the machine's threads, fed one scanline at a time (the work libspng
does; the scanlines are built beforehand with numpy, filtered and interlaced as asked, and not timed); Pillow's PNG encoder at
compress_level 6 goes beside it.  Bytes per frame are reported for the device's streams and for host zlib's.  The card's
name and power limit are read in the same run, and the kernel split comes from a separate torch.profiler pass.  One JSON line per workload; with --out, a summary in DIR/bench_pngsave.json."""
import argparse
import io
import json
import re
import os
import subprocess
import sys
import time
import zlib
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
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    base = (np.sin(xx / 37.0 + seed) + np.cos(yy / 53.0)) * 60 + 128
    if kind == "synthetic":
        a = (base // 24 * 24)[..., None].repeat(bands, 2)
        a[h // 3:h // 2] = 255
    else:
        a = base[..., None] + rng.normal(0, 6, (h, w, bands)).astype(np.float32)
    return np.clip(a, 0, 255).astype(np.uint8)


def batch(kind, n, h, w, bands, distinct=8):
    frames = [content(kind, h, w, bands, s) for s in range(min(n, distinct))]
    return np.stack([frames[i % len(frames)] for i in range(n)])


FILTERS = {"none": 0, "sub": 1, "up": 2, "avg": 3, "paeth": 4}
ADAM7 = ((0, 0, 8, 8), (4, 0, 8, 8), (0, 4, 4, 8), (2, 0, 4, 4), (0, 2, 2, 4), (1, 0, 2, 2), (0, 1, 1, 2))


def scanlines(a, filter, interlace):
    """the PNG scanlines of one 8-bit frame [h, w, bands] as a list of rows: Adam7 passes (PNG 2nd edition 8.2) or the frame,
    every row its filter type and its bytes filtered on the raw bytes (9.2)"""
    ft, bands, rows = FILTERS[filter], a.shape[2], []
    for x0, y0, dx, dy in (ADAM7 if interlace else ((0, 0, 1, 1),)):
        sub = a[y0::dy, x0::dx]
        if not sub.size:
            continue
        r = sub.reshape(sub.shape[0], -1).astype(np.int16)
        b, left, c = np.zeros_like(r), np.zeros_like(r), np.zeros_like(r)
        b[1:], left[:, bands:], c[1:, bands:] = r[:-1], r[:, :-bands], r[:-1, :-bands]
        if ft == 0:
            pred = 0
        elif ft == 1:
            pred = left
        elif ft == 2:
            pred = b
        elif ft == 3:
            pred = (left + b) >> 1
        else:
            p = left + b - c
            pa, pb, pc = np.abs(p - left), np.abs(p - b), np.abs(p - c)
            pred = np.where((pa <= pb) & (pa <= pc), left, np.where(pb <= pc, b, c))
        f = ((r - pred) & 255).astype(np.uint8)
        rows += [bytes([ft]) + row.tobytes() for row in f]
    return rows


def host_zlib(scans, threads):
    def one(rows):
        c = zlib.compressobj(6, zlib.DEFLATED, 15, 8, zlib.Z_DEFAULT_STRATEGY)
        return len(b"".join(c.compress(r) for r in rows) + c.flush())
    with ThreadPoolExecutor(threads) as ex:
        return list(ex.map(one, scans))


def host_pillow(frames, threads):
    def one(a):
        buf = io.BytesIO()
        PIL.fromarray(a if a.shape[2] > 1 else a[..., 0]).save(buf, "PNG", compress_level=6)
        return len(buf.getvalue())
    with ThreadPoolExecutor(threads) as ex:
        return list(ex.map(one, frames))


def timed(fn, reps, sync):
    fn()
    sync()
    best = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        sync()
        best.append(time.perf_counter() - t)
    return float(np.median(best))


def kernel_split(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        m = re.search(r"(deflate_\w+?_kernel|png_\w+?_kernel)", e.key)
        if m:
            out[m.group(1)] = round(out.get(m.group(1), 0.0) + e.device_time_total / 1000.0, 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    ap.add_argument("--small", type=int, default=2048)
    ap.add_argument("--big", type=int, default=16, help="large frames (0: skip that workload)")
    ap.add_argument("--filter", default="none", choices=sorted(FILTERS), help="every scanline's filter type")
    ap.add_argument("--interlace", action="store_true", help="Adam7 scanlines")
    args = ap.parse_args()
    opts = dict(filter=args.filter, interlace=args.interlace)
    tag = ("" if args.filter == "none" else "_" + args.filter) + ("_adam7" if args.interlace else "")
    import torch
    vb.init(0)
    name, power = card()
    threads = os.cpu_count() or 1
    sync = torch.cuda.synchronize
    results = []

    def device_save(frames):
        t = torch.from_numpy(frames).cuda()
        n, h, w, b = frames.shape
        return lambda: vb.pngsave_batch(None, 6, in_ptr=t.data_ptr(), shape=(n, h, w, b), **opts)

    for label, n, (h, w) in (("small", args.small, (256, 256)), ("big", args.big, (4096, 4096))):
        if n < 1:
            continue
        for bands in ((4, 3) if label == "small" else (3,)):
            for kind in ("synthetic", "photo"):
                frames = batch(kind, n, h, w, bands)
                run = device_save(frames)
                streams = run()
                for i in range(min(n, 8 if label == "small" else 1)):  # the host twin is serial: one large frame
                    assert streams[i] == vb.pngsave_host_twin(frames[i], 6, **opts), "device stream %d differs from the host twin" % i
                dev = timed(run, args.reps, sync)
                sub = frames[:max(1, min(n, 256 if label == "small" else 4))]
                scans = [scanlines(a, args.filter, args.interlace) for a in sub]
                hz_bytes = []
                hz = timed(lambda: hz_bytes.append(host_zlib(scans, threads)), 1, lambda: None) * n / len(sub)
                hp = timed(lambda: host_pillow(sub, threads), 1, lambda: None) * n / len(sub)
                r = {"workload": "%s_%s_%d%s" % (label, kind, bands, tag), "filter": args.filter, "interlace": args.interlace, "frames": n,
                     "shape": [h, w, bands], "gpu": name, "power_limit_max_sm": power,
                     "device_s": round(dev, 4), "device_frames_per_s": round(n / dev, 1),
                     "device_MB_per_s_in": round(frames.nbytes / dev / 1e6, 1),
                     "host_zlib_s": round(hz, 4), "host_zlib_frames_per_s": round(n / hz, 1),
                     "pillow_s": round(hp, 4), "pillow_frames_per_s": round(n / hp, 1), "host_threads": threads,
                     "ratio": round(sum(len(s) for s in streams) / frames.nbytes, 4),
                     "device_bytes_per_frame": round(sum(len(s) for s in streams) / n, 1),
                     "host_zlib_bytes_per_frame": round(float(np.mean(hz_bytes[-1])), 1),
                     "kernels_ms": kernel_split(run)}
                print(json.dumps(r), flush=True)
                results.append(r)
                del frames, streams
    # end to end: PNG streams -> run_png -> pngsave_batch
    if args.small < 4:
        return finish(args, results)
    src = batch("photo", args.small, 1024, 1024, 4, distinct=4)
    pngs = []
    for a in src[:4]:
        buf = io.BytesIO()
        PIL.fromarray(a).save(buf, "PNG", compress_level=6)
        pngs.append(buf.getvalue())
    streams = [pngs[i % 4] for i in range(args.small // 4)]
    plan = vb.ThumbnailPlan(1024, 1024, 4, 256)
    ow, oh = plan.out_width, plan.out_height
    out = torch.empty((len(streams), oh, ow, 4), dtype=torch.uint8, device="cuda")

    def e2e():
        plan.run_png(streams, out_ptr=out.data_ptr())
        return vb.pngsave_batch(None, 6, in_ptr=out.data_ptr(), shape=(len(streams), oh, ow, 4), **opts)
    got = e2e()
    th = out[:1].cpu().numpy()[0]
    assert got[0] == vb.pngsave_host_twin(th, 6, **opts)
    t = timed(e2e, args.reps, sync)
    r = {"workload": "e2e_png_thumbnail_png" + tag, "filter": args.filter, "interlace": args.interlace, "frames": len(streams),
         "in": [1024, 1024, 4], "out": [oh, ow, 4], "gpu": name,
         "power_limit_max_sm": power, "device_s": round(t, 4), "frames_per_s": round(len(streams) / t, 1)}
    print(json.dumps(r), flush=True)
    results.append(r)
    finish(args, results)


def finish(args, results):
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_pngsave.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()

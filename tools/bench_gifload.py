"""tools/bench_gifload.py -- GIF decode on the device (csrc/gif.cu) against libnsgif and Pillow on the host's own threads.

    python tools/bench_gifload.py [--reps R] [--threads T] [--out DIR]

Workloads (GIFs written by Pillow from a seed; a few distinct streams repeated to fill a batch):
    small   2048 streams of 256 x 256: static and 8-frame animations, synthetic (flat blocks, few colours) and photo-like
            (noise over smooth fields, quantized to 256 colours)
    big     16 static 4096 x 4096 frames, the same two contents
Reports, per workload: GIF frames decoded per second on the device (vb.gif_decode_batch of the last page into device
memory, so every frame of an animation is decoded and composed), libnsgif's own decode of the same streams through the
oracle built under oracle/_ref (nsgifload's copy over nsgif_frame_decode) on T host threads, Pillow's on T threads, and the
split between gif_lzw_kernel and gif_compose_kernel from a separate torch.profiler pass.  The card's name and power limit
are read in the same run.  One JSON line per workload; with --out, a summary in DIR/bench_gifload.json."""
import argparse
import ctypes as C
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
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the card's name still says what ran
        q = "unknown (%s)" % e
    return name, q


def content(kind, size, seed):
    rng = np.random.default_rng(seed)
    if kind == "synthetic":
        a = rng.integers(0, 256, (size // 16 + 1, size // 16 + 1, 3), dtype=np.uint8).repeat(16, 0).repeat(16, 1)[:size, :size]
        return PIL.fromarray(a).quantize(16)
    y, x = np.mgrid[0:size, 0:size].astype(np.float32)
    base = np.stack([128 + 100 * np.sin(x / (37 + 13 * c) + y / (53 + 7 * c) + c + seed) for c in range(3)], 2)
    a = np.clip(base + rng.normal(0, 12, base.shape), 0, 255).astype(np.uint8)
    return PIL.fromarray(a).quantize(256)


def gif_of(kind, size, frames, seed):
    ims = [content(kind, size, seed * 101 + k) for k in range(frames)]
    b = io.BytesIO()
    if frames == 1:
        ims[0].save(b, "GIF")
    else:
        ims[0].save(b, "GIF", save_all=True, append_images=ims[1:], duration=40, loop=0, disposal=1)
    return b.getvalue()


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


def host_timed(fn, reps):
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return float(np.median(t))


def kernel_split(batch, page, dev):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        vb.gif_decode_batch(batch, page, 1, out_ptr=dev.data_ptr())
        torch.cuda.synchronize()
    ms = {}
    for e in prof.key_averages():
        for k in ("gif_lzw_kernel", "gif_compose_kernel"):
            if k in e.key:
                ms[k] = ms.get(k, 0.0) + e.device_time_total / 1000.0
    return ms


def nsgif_lib():
    path = os.path.join(ROOT, "oracle", "_ref", "libnsgif_oracle.so")
    if not os.path.exists(path):
        return None
    L = C.CDLL(path)
    L.nsgif_oracle_load.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_int), C.c_char_p, C.c_size_t]
    return L


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    vb.init(0)
    name, limit = card()
    L = nsgif_lib()
    results = []
    work = [("small", kind, 256, frames, 2048) for frames in (1, 8) for kind in ("synthetic", "photo")] + \
           [("big", kind, 4096, 1, 16) for kind in ("synthetic", "photo")]
    for group, kind, size, frames, n in work:
        distinct = [gif_of(kind, size, frames, i) for i in range(min(n, 16))]
        batch = vb.StreamBatch([distinct[i % len(distinct)] for i in range(n)])
        w, h, bands, fc = vb.gif_geometry(distinct[0])
        page = fc - 1
        dev = torch.empty(n * w * h * bands, dtype=torch.uint8, device="cuda")
        t_dev = timed(lambda: vb.gif_decode_batch(batch, page, 1, out_ptr=dev.data_ptr()), args.reps)
        got = dev.view(n, h, w, bands)[n - 1].cpu().numpy()
        assert np.array_equal(got, vb.gif_decode_host_twin(batch.streams[n - 1], page, 1)), "device decode differs from the host twin"
        split = kernel_split(batch, page, dev)
        pool = ThreadPoolExecutor(args.threads)
        t_ns = None
        if L is not None:
            def ns_one(s):
                info = (C.c_int * 5)()
                out = np.empty((h, w, bands), np.uint8)
                if L.nsgif_oracle_load(s, len(s), page, 1, out.ctypes.data, info, None, 0):
                    raise RuntimeError("libnsgif failed")
            t_ns = host_timed(lambda: list(pool.map(ns_one, batch.streams)), max(1, args.reps // 2))

        def pil_one(s):
            im = PIL.open(io.BytesIO(s))
            im.seek(page)
            im.convert("RGBA" if bands == 4 else "RGB").tobytes()
        t_pil = host_timed(lambda: list(pool.map(pil_one, batch.streams)), max(1, args.reps // 2))
        pool.shutdown()
        gif_frames = n * fc
        r = {"workload": "%s_%s_%dframe" % (group, kind, frames), "streams": n, "size": size, "frames_per_stream": fc, "bands": bands,
             "compressed_MB": round(batch.nbytes / 1e6, 2),
             "device_frames_per_s": round(gif_frames / t_dev[0], 1), "device_s": [round(v, 4) for v in t_dev],
             "lzw_ms": round(split.get("gif_lzw_kernel", 0.0), 2), "compose_ms": round(split.get("gif_compose_kernel", 0.0), 2),
             "libnsgif_frames_per_s": round(gif_frames / t_ns, 1) if t_ns else "not measured (oracle/_ref not built)",
             "pillow_frames_per_s": round(gif_frames / t_pil, 1), "host_threads": args.threads,
             "gpu": name, "power_limit_max_sm_clock": limit}
        print(json.dumps(r), flush=True)
        results.append(r)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_gifload.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()

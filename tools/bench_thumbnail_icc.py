"""tools/bench_thumbnail_icc.py -- the colour-managed thumbnail (vb200_thumbnail_plan_set_icc) against the plain one.

    python tools/bench_thumbnail_icc.py [--frames 512] [--steps 5]

Prints one JSON line per workload, each with the card name and power limit read in the same run:
  (a) device-resident 4096 x 4096 RGBA frames -> 512, each tagged with tests/golden/profiles/p3.icm, output sRGB.icm;
  (b) the same frames with colour management off, timed alternately with (a) in this process;
  (c) P3-tagged JPEG streams through run_jpeg (decode + thumbnail), with and without colour management.
frames/s is over whole batch calls timed with CUDA events.  icc_stage_ms is the median over separate calls of CUDA events
recorded around the stage's icc_frames_kernel launches inside the library (env VB200_ICC_TIMING, vb200_debug_icc_stage_ms),
with no profiler attached; icc_stage_gbps is icc_stage_bytes over that time.  icc_stage_bytes are the stage's algorithmic
bytes per batch (the thumbnail frames read, the colour-managed frames written, the job table and index array)."""
import argparse
import ctypes
import io
import json
import os
import subprocess
import sys

import numpy as np

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


def timed(fn, steps):
    import torch
    out = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return float(np.median(out))


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--jpeg-frames", type=int, default=64)
    args = ap.parse_args()
    vb.init(0)
    prof = lambda n: open(os.path.join(ROOT, "tests", "golden", "profiles", n), "rb").read()
    srgb, p3 = prof("sRGB.icm"), prof("p3.icm")
    info = card()
    n, W = args.frames, 4096
    g = torch.Generator(device="cuda").manual_seed(1)
    frames = torch.randint(0, 256, (n, W, W, 4), dtype=torch.uint8, device="cuda", generator=g)
    plain = vb.ThumbnailPlan(W, W, 4, 512)
    icc = vb.ThumbnailPlan(W, W, 4, 512)
    icc.set_icc(srgb, builtin_profiles={"srgb": srgb})
    out = torch.empty((n, icc.out_height, icc.out_width, 4), dtype=torch.uint8, device="cuda")
    emb = [p3] * n
    run_plain = lambda: plain.run_device(frames.data_ptr(), out.data_ptr(), n)
    run_icc = lambda: icc.run_device(frames.data_ptr(), out.data_ptr(), n, embedded=emb)
    run_plain(), run_icc()
    torch.cuda.synchronize()
    ta, tb = [], []
    for _ in range(args.steps):           # (a) and (b) alternated
        ta.append(timed(run_icc, 1))
        tb.append(timed(run_plain, 1))
    ma, mb = float(np.median(ta)), float(np.median(tb))
    os.environ["VB200_ICC_TIMING"] = "1"
    vb.lib().vb200_debug_icc_stage_ms.restype = ctypes.c_float
    stage = []
    for _ in range(args.steps):
        run_icc()
        stage.append(float(vb.lib().vb200_debug_icc_stage_ms()))
    del os.environ["VB200_ICC_TIMING"]
    ms_stage = float(np.median(stage))
    px = icc.out_width * icc.out_height
    stage_bytes = n * px * (4 + icc.out_bands) + n * 4 + 4096
    base = {"frame": "%dx%dx4 u8 -> %dx%d" % (W, W, icc.out_width, icc.out_height), "frames": n, "steps": args.steps, **info}
    print(json.dumps({"workload": "a: thumbnail + ICC (p3 -> sRGB), device-resident", "ms_per_batch": ma, "frames_per_s": n / ma * 1e3,
                      "icc_stage_ms": ms_stage, "icc_stage_bytes": stage_bytes,
                      "icc_stage_gbps": stage_bytes / ms_stage / 1e6, "calls_minus_plain_ms": ma - mb, "kernel": plain.kernel, **base}))
    print(json.dumps({"workload": "b: thumbnail, ICC off, device-resident", "ms_per_batch": mb, "frames_per_s": n / mb * 1e3,
                      "bytes_per_frame": plain.bytes_per_frame, "kernel": plain.kernel, **base}))
    del frames, out
    torch.cuda.empty_cache()
    # (c) JPEG streams carrying the P3 profile
    from PIL import Image as PIL
    rng = np.random.default_rng(2)
    a = np.clip(rng.normal(128, 40, (2048, 2048, 3)), 0, 255).astype(np.uint8)
    b = io.BytesIO()
    PIL.fromarray(a).save(b, "JPEG", quality=85, icc_profile=p3)
    streams = vb.JpegBatch([b.getvalue()] * args.jpeg_frames)
    shrink = vb.thumbnail_jpegshrink(2048, 2048, 256)
    w, h, bands = vb.jpeg_geometry(streams, shrink)
    for on in (True, False):
        plan = vb.ThumbnailPlan(w, h, bands, 256)
        if on:
            plan.set_icc(srgb, builtin_profiles={"srgb": srgb})
        res = torch.empty((streams.n, plan.out_height, plan.out_width, plan.out_bands), dtype=torch.uint8, device="cuda")
        go = lambda: plan.run_jpeg(streams, shrink, out_ptr=res.data_ptr())
        go()
        ms = timed(go, args.steps)
        print(json.dumps({"workload": "c: run_jpeg 2048x2048 P3-tagged streams -> 256, ICC %s" % ("on" if on else "off"),
                          "ms_per_batch": ms, "frames_per_s": streams.n / ms * 1e3, "frames": streams.n, "shrink_on_load": shrink,
                          "steps": args.steps, **info}))


if __name__ == "__main__":
    main()

"""tools/bench_thumbnail_linear_icc.py -- the colour-managed linear thumbnail (vb200_thumbnail_plan_set_linear_icc) against the
plain linear one.

    python tools/bench_thumbnail_linear_icc.py [--frames 64] [--steps 5]

Prints one JSON line per workload, each with the card name and power limit read in the same run:
  (a) device-resident 4096 x 4096 RGBA frames -> 512, linear, each tagged with tests/golden/profiles/p3.icm, output sRGB.icm:
      the import in the V kernel, the export in the H kernel (branch I);
  (b) the same frames, linear, no colour management, timed alternately with (a) in this process.
vh_ms is the median over separate batch calls of CUDA events recorded inside the library from before the first linear_v launch
to after the last linear_h launch of the call (env VB200_LINEAR_TIMING, vb200_debug_linear_thumb_ms), no profiler attached.
call_ms is the median of CUDA events around whole calls, which also holds the host's per-batch work (profile selection, job
table upload, scratch allocation).  bytes_per_frame is the algorithmic figure (frame in + thumbnail out)."""
import argparse
import ctypes
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


def timed(fn):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()
    vb.init(0)
    prof = lambda n: open(os.path.join(ROOT, "tests", "golden", "profiles", n), "rb").read()
    srgb, p3 = prof("sRGB.icm"), prof("p3.icm")
    info = card()
    n, W = args.frames, 4096
    g = torch.Generator(device="cuda").manual_seed(1)
    frames = torch.randint(0, 256, (n, W, W, 4), dtype=torch.uint8, device="cuda", generator=g)
    plain = vb.ThumbnailPlan(W, W, 4, 512, linear=True)
    icc = vb.ThumbnailPlan(W, W, 4, 512, linear=True)
    icc.set_linear_icc(srgb, builtin_profiles={"srgb": srgb})
    out = torch.empty((n, icc.out_height, icc.out_width, icc.out_bands), dtype=torch.uint8, device="cuda")
    emb = [p3] * n
    vb.set_stream(torch.cuda.current_stream().cuda_stream)
    run_plain = lambda: plain.run_device(frames.data_ptr(), out.data_ptr(), n)
    run_icc = lambda: icc.run_device(frames.data_ptr(), out.data_ptr(), n, embedded=emb)
    run_plain(), run_icc()
    torch.cuda.synchronize()
    ta, tb = [], []
    for _ in range(args.steps):           # (a) and (b) alternated
        ta.append(timed(run_icc))
        tb.append(timed(run_plain))
    ma, mb = float(np.median(ta)), float(np.median(tb))
    os.environ["VB200_LINEAR_TIMING"] = "1"
    vb.lib().vb200_debug_linear_thumb_ms.restype = ctypes.c_float
    va, vbb = [], []
    for _ in range(args.steps):           # (a) and (b) alternated, V + H launches only
        run_icc()
        va.append(float(vb.lib().vb200_debug_linear_thumb_ms()))
        run_plain()
        vbb.append(float(vb.lib().vb200_debug_linear_thumb_ms()))
    del os.environ["VB200_LINEAR_TIMING"]
    vha, vhb = float(np.median(va)), float(np.median(vbb))
    base = {"frame": "%dx%dx4 u8 -> %dx%d linear" % (W, W, icc.out_width, icc.out_height), "frames": n, "steps": args.steps,
            "kernel": plain.kernel, "bytes_per_frame": plain.bytes_per_frame, **info}
    print(json.dumps({"workload": "a: linear thumbnail + ICC (p3 import -> sRGB export), device-resident", "vh_ms": vha,
                      "vh_ms_per_frame": vha / n, "call_ms": ma, "frames_per_s": n / ma * 1e3,
                      "vh_minus_plain_ms_per_frame": (vha - vhb) / n, **base}))
    print(json.dumps({"workload": "b: linear thumbnail, ICC off, device-resident", "vh_ms": vhb, "vh_ms_per_frame": vhb / n,
                      "call_ms": mb, "frames_per_s": n / mb * 1e3, **base}))


if __name__ == "__main__":
    main()

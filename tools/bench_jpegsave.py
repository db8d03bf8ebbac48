"""tools/bench_jpegsave.py -- the device JPEG encoder (vb200_jpegsave_batch_opts) with vips_jpegsave's entropy options.

    python tools/bench_jpegsave.py [--frames 512] [--size 512] [--steps 10] [--cpu-frames 64]

512 seeded, photo-like 512 x 512 RGB frames resident on the device, encoded into device memory at Q 75 and Q 90 in six
configurations: default, optimize_coding, restart_interval = one MCU row, both, and progressive (interlace) without and
with restart_interval = one MCU row.  Each batch call is timed with CUDA
events after a warm-up call; ms is the median over --steps calls.  Per configuration it prints ms per batch, frames/s,
the kernel launches one call makes (vb.launch_count) and the mean stream size relative to the default configuration.
Beside it, Pillow (libjpeg-turbo) with the same options over the host's cores, one frame per task, as the CPU
comparison.  The card name and power limit are read in the same run.  One JSON line per (Q, configuration).
"""
import argparse
import ctypes as C
import io
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
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


def pil_one(args):
    from PIL import Image
    a, q, opt, r, il = args
    b = io.BytesIO()
    kw = {"optimize": True} if opt else {}
    if r:
        kw["restart_marker_blocks"] = r
    if il:
        kw["progressive"] = True
    Image.fromarray(a).save(b, "JPEG", quality=q, subsampling=2 if q < 90 else 0, **kw)
    return len(b.getvalue())


def main():
    import torch
    from test_jpeg import synth
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--cpu-frames", type=int, default=64)
    args = ap.parse_args()
    vb.init(0)
    info = card()
    n, s = args.frames, args.size
    host = np.stack([synth(s, s, seed=i) for i in range(n)])
    frames = torch.from_numpy(host).cuda()
    stride = s * s * 3 * 2 + 4096
    out = torch.empty((n, stride), dtype=torch.uint8, device="cuda")
    lens = (C.c_size_t * n)()
    L = vb.lib()
    pool = ProcessPoolExecutor(os.cpu_count() or 1)

    def call(opts):
        vb._check(L.vb200_jpegsave_batch_opts(C.c_void_p(frames.data_ptr()), vb.DEVICE, s * 3, s * s * 3, n, s, s, 3, C.byref(opts),
                                              C.c_void_p(out.data_ptr()), vb.DEVICE, stride, lens))

    for q in (75, 90):
        mcu = 16 if q < 90 else 8
        row = (s + mcu - 1) // mcu
        base_bytes = None
        for name, opt, r, il in (("default", 0, 0, 0), ("optimize", 1, 0, 0), ("restart_row", 0, row, 0), ("optimize+restart_row", 1, row, 0),
                                 ("interlace", 0, 0, 1), ("interlace+restart_row", 0, row, 1)):
            opts = vb.JpegSaveOptions(q, 0, opt, r, il)
            call(opts)                                   # warm-up
            torch.cuda.synchronize()
            before = vb.launch_count()
            call(opts)
            launches = vb.launch_count() - before
            mean_bytes = float(np.mean(list(lens)))
            if base_bytes is None:
                base_bytes = mean_bytes
            times = []
            for _ in range(args.steps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                call(opts)
                b.record()
                b.synchronize()
                times.append(a.elapsed_time(b))
            ms = float(np.median(times))
            cpu_n = min(args.cpu_frames, n)
            work = [(host[i], q, opt, r, il) for i in range(cpu_n)]
            list(pool.map(pil_one, work[:4]))            # start the workers
            t0 = time.perf_counter()
            list(pool.map(pil_one, work))
            cpu_fps = cpu_n / (time.perf_counter() - t0)
            print(json.dumps(dict(info, workload="jpegsave %d x %dx%d RGB, device in/out" % (n, s, s), Q=q, config=name,
                                  optimize_coding=opt, restart_interval=r, interlace=il, ms_per_batch=round(ms, 3), frames_per_s=round(n / ms * 1e3, 1),
                                  launches_per_call=launches, mean_bytes=round(mean_bytes, 1),
                                  bytes_vs_default=round(mean_bytes / base_bytes, 4), pillow_frames_per_s=round(cpu_fps, 1),
                                  pillow_workers=os.cpu_count())), flush=True)
    pool.shutdown()


if __name__ == "__main__":
    main()

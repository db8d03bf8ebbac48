"""tools/bench_webp_thumbnail.py -- WebP thumbnails on the device: shrink-on-load (ThumbnailPlan.run_webp, libwebp's scaled
decode as vips_thumbnail asks for it) against a full-size decode followed by the plan, over the same streams.

    python tools/bench_webp_thumbnail.py [--batch N] [--reps R] [--out DIR]

Workload: batches of seeded 2048 x 1536 quality-80 streams (Pillow's encoder, a few distinct ones repeated) to 256-pixel
thumbnails, the output left on the device.  Both paths are warmed up once and timed as the median of --reps runs; each
path's device time is also split per WebP kernel (the library's CUDA events, VB200_WEBP_TIMING, over one batch: the
"rgb" slot is the scaled output kernel on the shrink-on-load path).  The card's name and power limit are read in the same
run.  One JSON line per path; with --out, a summary in DIR/bench_webp_thumbnail.json."""
import argparse
import json
import os
import sys

ROOT = __file__.rsplit("/tools/", 1)[0]
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import libvips_b200 as vb  # noqa: E402
from bench_webpload import card, kernel_split, photo, timed, webp  # noqa: E402

W, H, TARGET = 2048, 1536, 256


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    vb.init(0)
    name, power = card()
    print(json.dumps({"card": name, "power_limit": power}), flush=True)
    n = args.batch
    distinct = [webp(photo(H, W, i), 80) for i in range(4)]
    batch = vb.StreamBatch([distinct[i % len(distinct)] for i in range(n)])
    scale, sw, sh = vb.thumbnail_webp_scale(W, H, TARGET)
    scaled_plan = vb.ThumbnailPlan(sw, sh, 3, TARGET)
    full_plan = vb.ThumbnailPlan(W, H, 3, TARGET)
    out = torch.empty(n * full_plan.out_frame_bytes, dtype=torch.uint8, device="cuda")
    frames = torch.empty(n * W * H * 3, dtype=torch.uint8, device="cuda")

    def full():
        vb.webp_decode_batch(batch, out_ptr=frames.data_ptr())
        full_plan.run_device(frames.data_ptr(), out.data_ptr(), n)

    paths = [("shrink_on_load", lambda: scaled_plan.run_webp(batch, scale, out_ptr=out.data_ptr()), (sw, sh)),
             ("full_decode_then_plan", full, (W, H))]
    results = []
    for label, fn, decoded in paths:
        t = timed(fn, args.reps, torch.cuda.synchronize)
        r = {"path": label, "frames": n, "source": [W, H], "decoded": list(decoded), "scale": scale, "thumbnail": [scaled_plan.out_width,
             scaled_plan.out_height], "frames_per_s": n / t, "webp_kernel_ms_per_batch": kernel_split(fn)}
        print(json.dumps(r), flush=True)
        results.append(r)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_webp_thumbnail.json"), "w") as f:
            json.dump({"card": name, "power_limit": power, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()

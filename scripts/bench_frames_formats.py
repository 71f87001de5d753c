"""Camera frames in other pixel formats: the fused convert-and-resize kernel per format against RGB, the full-size conversion, and the
frames-to-key-points step with NV12 frames.

    python scripts/bench_frames_formats.py [--steps 20] [--launches 200] [--rounds 2] [--out result.json]

1. h3d_resize_frames_fmt (normalize = 1, into 240x320) at B = 32 for 480x640, 720x1280, 1080x1920 and 2160x3840 frames, every format,
   the formats interleaved in one process (--rounds passes over them; the best pass is kept): CUDA events over --launches launches
   after warm-up.  Bytes = the frames read once in the format's layout + the float32 output written, computed from the shapes, against
   the H100 SXM data-sheet 3.35 TB/s.
2. h3d_convert_frames at B = 32, 1080p, every format: bytes = the frames read + the RGB frames written.
3. B = 32 frames of 1080p to key-points through FrameRunner.stream, host frames in, wall clock over --steps steps:
   (a) NV12 frames converted to RGB on the host with cv2.cvtColor, then the RGB runner (skipped without OpenCV);
   (b) RGB frames, the RGB runner;
   (c) NV12 frames, FrameRunner(pixel_format="nv12").
The card's name, power limit and max SM clock are read in the same run.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench_frames import HBM_BYTES_PER_S, card  # noqa: E402
from hand3d_b200 import frames as FR  # noqa: E402
from hand3d_b200 import runtime  # noqa: E402
from hand3d_b200 import weights as Wt  # noqa: E402

FORMATS = ["rgb", "bgr", "nv12", "i420", "yuyv"]


def _events(fn, launches):
    for _ in range(20):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000.0 / launches


def _row(what, fmt, B, H, W, us, read, written):
    floor_us = (read + written) / HBM_BYTES_PER_S * 1e6
    return {"what": what, "format": fmt, "frames": "%dx%dx%d" % (B, H, W), "us": round(us, 2), "bytes_read": read,
            "GB_per_s": round((read + written) / us / 1e3, 1), "hbm_floor_us": round(floor_us, 2), "share_of_floor": round(floor_us / us, 3)}


def kernel_times(ctx, B, H, W, launches, rounds):
    g = torch.Generator(device="cuda").manual_seed(1)
    frames = {f: torch.randint(0, 256, (B,) + FR.frame_shape(f, H, W), dtype=torch.uint8, device="cuda", generator=g) for f in FORMATS}
    out = torch.empty((B, 240, 320, 3), dtype=torch.float32, device="cuda")
    best = {}
    for _ in range(rounds):
        for f in FORMATS:
            us = _events(lambda: ctx.resize_frames(frames[f], 240, 320, True, out=out, pixel_format=f), launches)
            best[f] = min(us, best.get(f, us))
    rows = [_row("resize_frames_fmt", f, B, H, W, best[f], frames[f].numel(), out.numel() * 4) for f in FORMATS]
    for r in rows:
        r["vs_rgb"] = round(r["us"] / best["rgb"], 3)
    return rows


def convert_times(ctx, B, H, W, launches):
    g = torch.Generator(device="cuda").manual_seed(2)
    rgb = torch.empty((B, H, W, 3), dtype=torch.uint8, device="cuda")
    rows = []
    for f in FORMATS:
        fr = torch.randint(0, 256, (B,) + FR.frame_shape(f, H, W), dtype=torch.uint8, device="cuda", generator=g)
        us = _events(lambda: ctx.convert_frames(fr, f, out=rgb), launches)
        rows.append(_row("convert_frames", f, B, H, W, us, fr.numel(), rgb.numel()))
    return rows


def stream_ms(runner, batches, steps):
    for _ in runner.stream(batches(i) for i in range(3)):
        pass
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = 0
    for _ in runner.stream(batches(i) for i in range(steps)):
        n += 1
    return (time.perf_counter() - t0) * 1000.0 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_frames_formats.py needs a CUDA device")
    ctx = runtime.Context(0)
    ctx.load_weights(Wt.synthetic_weights(0))
    res = {"card": card(), "kernel": [], "convert": [], "step_1080p_b32": {}}
    print(json.dumps(res["card"]), flush=True)
    for H, W in [(480, 640), (720, 1280), (1080, 1920), (2160, 3840)]:
        for r in kernel_times(ctx, 32, H, W, args.launches, args.rounds):
            res["kernel"].append(r)
            print(json.dumps(r), flush=True)
    for r in convert_times(ctx, 32, 1080, 1920, args.launches):
        res["convert"].append(r)
        print(json.dumps(r), flush=True)

    B, H, W = 32, 1080, 1920
    nv12 = [np.stack([np.random.default_rng(100 * i + b).integers(0, 256, FR.frame_shape("nv12", H, W), dtype=np.uint8) for b in range(B)])
            for i in range(2)]
    rgb = [np.stack([np.random.default_rng(300 * i + b).integers(0, 256, (H, W, 3), dtype=np.uint8) for b in range(B)]) for i in range(2)]
    steps = res["step_1080p_b32"]
    runner = FR.FrameRunner(ctx, B, (H, W))
    try:
        import cv2
    except ImportError:
        cv2 = None
    if cv2 is None:
        print("(a) not run: OpenCV is not installed", flush=True)
        steps["a_host_cvtcolor_then_rgb"] = None
    else:
        steps["a_host_cvtcolor_then_rgb"] = stream_ms(
            runner, lambda i: np.stack([cv2.cvtColor(f, cv2.COLOR_YUV2RGB_NV12) for f in nv12[i % 2]]), args.steps)
    steps["b_rgb"] = stream_ms(runner, lambda i: rgb[i % 2], args.steps)
    del runner
    ctx.release_graphs()
    runner = FR.FrameRunner(ctx, B, (H, W), pixel_format="nv12")
    steps["c_nv12"] = stream_ms(runner, lambda i: nv12[i % 2], args.steps)
    del runner
    ctx.release_graphs()
    for k, v in list(steps.items()):
        if v is not None:
            steps[k] = {"ms_per_step": round(v, 2), "frames_per_s": round(B * 1000.0 / v, 1)}
    print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

"""Camera frames: times h3d_resize_frames alone and the frames-to-key-points step three ways.

    python scripts/bench_frames.py [--steps 20] [--launches 200] [--out result.json]

1. The resize kernel (normalize = 1, the pipeline's float32 input) at B = 32 for 480x640, 720x1280, 1080x1920 and 2160x3840 frames
   -> 240x320: CUDA events over --launches launches after warm-up; bytes = the frames read once + the float32 output written,
   computed from the shapes, against the H100 SXM data-sheet 3.35 TB/s.
2. B = 32 frames of 1080p to key-points, host frames in, wall clock over --steps steps ending in a synchronise:
   (a) Pillow resize + normalisation on the host, float32 upload, then the captured pipeline;
   (b) uint8 upload, then the device resize and the captured pipeline, in series on one stream;
   (c) FrameRunner.stream: the upload of batch i + 1 overlaps the replay of batch i.
The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hand3d_b200 import frames as FR  # noqa: E402
from hand3d_b200 import runtime  # noqa: E402
from hand3d_b200 import weights as Wt  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip().splitlines()[0]
    except Exception as e:      # the number is still reported, with the reason the power limit is missing
        info["power_limit_and_max_sm_clock"] = "unavailable (%s)" % e
    return info


def time_kernel(ctx, B, H, W, launches):
    g = torch.Generator(device="cuda").manual_seed(1)
    fr = torch.randint(0, 256, (B, H, W, 3), dtype=torch.uint8, device="cuda", generator=g)
    out = torch.empty((B, 240, 320, 3), dtype=torch.float32, device="cuda")
    for _ in range(20):
        ctx.resize_frames(fr, 240, 320, True, out=out)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        ctx.resize_frames(fr, 240, 320, True, out=out)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1000.0 / launches
    read, written = B * H * W * 3, B * 240 * 320 * 3 * 4
    floor_us = (read + written) / HBM_BYTES_PER_S * 1e6
    return {"frames": "%dx%dx%d" % (B, H, W), "us": round(us, 2), "GB_per_s": round((read + written) / us / 1e3, 1),
            "hbm_floor_us": round(floor_us, 2), "share_of_floor": round(floor_us / us, 3)}


def pil_prepare(frames):
    try:
        from PIL import Image
    except ImportError:
        return None
    return np.stack([(np.asarray(Image.fromarray(f).resize((320, 240), Image.BILINEAR)).astype(np.float64) / 255.0 - 0.5).astype(np.float32)
                     for f in frames])


def time_steps(fn, steps, warmup=3):
    for i in range(warmup):
        fn(i)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        fn(i)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1000.0 / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_frames.py needs a CUDA device")
    ctx = runtime.Context(0)
    ctx.load_weights(Wt.synthetic_weights(0))
    res = {"card": card(), "kernel": [], "step_1080p_b32": {}}
    for H, W in [(480, 640), (720, 1280), (1080, 1920), (2160, 3840)]:
        res["kernel"].append(time_kernel(ctx, 32, H, W, args.launches))
        print(json.dumps(res["kernel"][-1]), flush=True)

    B, H, W = 32, 1080, 1920
    host = [np.stack([np.random.default_rng(100 * i + b).integers(0, 256, (H, W, 3), dtype=np.uint8) for b in range(B)]) for i in range(2)]
    hs = torch.tensor([[1.0, 0.0]] * B, dtype=torch.float32, device="cuda")
    image = torch.empty((B, 240, 320, 3), dtype=torch.float32, device="cuda")
    image_pinned = torch.empty(image.shape, dtype=torch.float32).pin_memory()
    frames_dev = torch.empty((B, H, W, 3), dtype=torch.uint8, device="cuda")
    frames_pinned = torch.empty(frames_dev.shape, dtype=torch.uint8).pin_memory()
    ctx.resize_frames(frames_dev, 240, 320, True, out=image)
    replay, _ = ctx.capture_pipeline(image, hs, True, outputs="keypoints")
    steps = res["step_1080p_b32"]

    if pil_prepare(host[0][:1]) is None:
        print("(a) not run: Pillow is not installed", flush=True)
        steps["a_pillow_host"] = None
    else:
        def step_a(i):
            image_pinned.copy_(torch.from_numpy(pil_prepare(host[i % 2])))
            image.copy_(image_pinned, non_blocking=True)
            replay()
        steps["a_pillow_host"] = time_steps(step_a, args.steps)

    def step_b(i):
        frames_pinned.copy_(torch.from_numpy(host[i % 2]))
        frames_dev.copy_(frames_pinned, non_blocking=True)
        ctx.resize_frames(frames_dev, 240, 320, True, out=image)
        replay()
    steps["b_device_resize_serial"] = time_steps(step_b, args.steps)
    ctx.release_graphs()
    del replay

    runner = FR.FrameRunner(ctx, B, (H, W))
    for _ in runner.stream(host[i % 2] for i in range(3)):
        pass
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = 0
    for _ in runner.stream(host[i % 2] for i in range(args.steps)):
        n += 1
    steps["c_frame_runner_overlap"] = (time.perf_counter() - t0) * 1000.0 / n
    for k, v in list(steps.items()):
        if v is not None:
            steps[k] = {"ms_per_step": round(v, 2), "frames_per_s": round(B * 1000.0 / v, 1)}
    print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

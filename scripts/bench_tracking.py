"""Tracking across camera frames: what a track step (no HandSegNet) saves against a detect step.

    python scripts/bench_tracking.py [--replays 200] [--steps 60] [--out result.json]

1. Single-slot latency at 240x320 (run.py's network input): a detect step and a track step of Context.track_step, each captured into
   a CUDA graph; CUDA events over --replays replays, in three alternating rounds (the median is reported).
2. FrameRunner frames/s on 1080p uint8 host frames at B = 1 and B = 32: without tracking, and with track=True for redetect_every in
   {1, 10, 30, None} (no score test, so only the fall-backs lose a slot); wall clock over --steps batches of FrameRunner.stream after
   a warm-up, ending in the read-back of the last batch.
3. The update kernel's time from torch.profiler (a run of its own) over the track-step replays.
Both for bf16x3 and fp16.  The card's name and power limit are read in the same run.
"""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hand3d_b200 import runtime  # noqa: E402
from hand3d_b200 import weights as Wt  # noqa: E402
from hand3d_b200.frames import FrameRunner  # noqa: E402


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip().splitlines()[0]
    except Exception as e:      # the number is still reported, with the reason the power limit is missing
        info["power_limit_and_max_sm_clock"] = "unavailable (%s)" % e
    return info


def capture(ctx, image, hs, state, detect):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):       # warm-up outside capture: plans, packed weights
        ctx.track_step(image, hs, state, detect, outputs="keypoints")
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ctx.track_step(image, hs, state, detect, outputs="keypoints")
    ctx._graphs_captured = getattr(ctx, "_graphs_captured", 0) + 1
    return g


def time_replays(g, n):
    for _ in range(10):
        g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000.0 / n


def single_slot(ctx, replays):
    image = torch.from_numpy(Wt.synthetic_blob_images(1, 240, 320, seed=3)).cuda()
    hs = torch.tensor([[1.0, 0.0]], dtype=torch.float32, device="cuda")
    state = runtime.TrackState(1)
    graphs = {"detect": capture(ctx, image, hs, state, True), "track": capture(ctx, image, hs, state, False)}
    rounds = {k: [] for k in graphs}
    for _ in range(3):
        for k, g in graphs.items():
            rounds[k].append(time_replays(g, replays))
    out = {k + "_step_us": round(float(np.median(v)), 1) for k, v in rounds.items()}
    out["track_over_detect"] = round(out["track_step_us"] / out["detect_step_us"], 3)
    # the update kernel, profiled in a run of its own
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(50):
            graphs["track"].replay()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "track_update_kernel" in e.name]
    out["update_kernel_us_b1"] = round(sum(e.device_time for e in ev) / max(1, len(ev)), 2) if ev else None
    del graphs
    ctx.release_graphs()
    return out


def update_kernel_b32(ctx):
    B = 32
    rng = np.random.default_rng(0)
    m = torch.from_numpy(rng.normal(0, 1, (B, 32, 32, 21)).astype(np.float32)).cuda()
    uv = torch.from_numpy(rng.integers(0, 256, (B, 21, 2)).astype(np.int32)).cuda()
    c = torch.full((B, 2), 160.0, device="cuda")
    s = torch.ones(B, device="cuda")
    st = runtime.TrackState(B)
    for _ in range(10):
        ctx.track_update(m, uv, c, s, st)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(50):
            ctx.track_update(m, uv, c, s, st)
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "track_update_kernel" in e.name]
    return round(sum(e.device_time for e in ev) / max(1, len(ev)), 2) if ev else None


def frames_per_s(ctx, B, host, steps, **kw):
    runner = FrameRunner(ctx, B, host[0].shape[1:3], **kw)
    try:
        for _ in runner.stream(host[i % 2] for i in range(3)):   # warm-up: steps 0-2 (step 0 detects)
            pass
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        n = 0
        for _ in runner.stream(host[i % 2] for i in range(steps)):
            n += 1
        dt = time.perf_counter() - t0
    finally:
        del runner
        ctx.release_graphs()
        gc.collect()
        torch.cuda.empty_cache()
    return round(B * n / dt, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replays", type=int, default=200)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--batches", default="1,32")
    ap.add_argument("--precisions", default="bf16x3,fp16")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tracking.py needs a CUDA device")
    ctx = runtime.Context(0)
    ctx.load_weights(Wt.synthetic_weights(0))
    res = {"card": card(), "results": {}}
    print(json.dumps(res["card"]), flush=True)
    H, W = 1080, 1920
    for prec in args.precisions.split(","):
        ctx.set_precision(prec)
        r = res["results"][prec] = {"single_slot_240x320": single_slot(ctx, args.replays), "update_kernel_us_b32": update_kernel_b32(ctx)}
        print(prec, json.dumps(r), flush=True)
        for B in [int(b) for b in args.batches.split(",")]:
            host = [np.stack([np.random.default_rng(100 * i + b).integers(0, 256, (H, W, 3), dtype=np.uint8) for b in range(B)])
                    for i in range(2)]
            row = r["frame_runner_1080p_b%d_frames_per_s" % B] = {"no_tracking": frames_per_s(ctx, B, host, args.steps)}
            for every in (1, 10, 30, None):
                row["track_redetect_%s" % every] = frames_per_s(ctx, B, host, args.steps, track=True, redetect_every=every)
            print(prec, B, json.dumps(row), flush=True)
    print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

"""Per-slot re-detection (h3d_track_step_slots): what a step costs when k of B slots re-detect, against a track step and a detect step.

    python scripts/bench_track_slots.py [--replays 100] [--steps 60] [--out result.json]

1. Steps at B = 32 slots of 240x320 (run.py's network input), min_score None: h3d_track_step with detect = 0 and detect = 1, and
   h3d_track_step_slots with k in {0, 1, 2, 4, 8, 16, 32} slots forced (the first k).  Every step is captured into a CUDA graph that
   first clears the state's lost flags (one memset in every graph, so that exactly the k forced slots re-detect); CUDA events over
   --replays replays, the graphs alternating in three rounds (the median is reported).  The prediction
   track + (k / 32) (detect - track) is printed beside each measured slots step.
2. FrameRunner frames/s on 1080p uint8 host frames at B = 32: detect="batch" with redetect_every=1 (what one lost slot per step
   costs that policy: every step detects) and redetect_every=None, against detect="slots" with redetect_every=32 (one slot forced per
   step) and None; wall clock over --steps batches of FrameRunner.stream after a warm-up.  The slots runs also report the mean number of
   slots re-detected per step (fall-backs on the noise frames can add to the forced one).
Both for bf16x3 and fp16.  The card's name and power limit are read in the same run.
"""
import argparse
import gc
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_tracking import card, time_replays  # noqa: E402
from hand3d_b200 import runtime  # noqa: E402
from hand3d_b200 import weights as Wt  # noqa: E402
from hand3d_b200.frames import FrameRunner  # noqa: E402

KS = (0, 1, 2, 4, 8, 16, 32)


def capture(ctx, fn, state):
    def body():
        state.lost.zero_()
        fn()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):       # warm-up outside capture: plans, packed weights
        body()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        body()
    ctx._graphs_captured = getattr(ctx, "_graphs_captured", 0) + 1
    return g


def steps(ctx, B, replays):
    image = torch.from_numpy(Wt.synthetic_blob_images(B, 240, 320, seed=3)).cuda()
    hs = torch.tensor([[1.0, 0.0]] * B, dtype=torch.float32, device="cuda")
    state = runtime.TrackState(B)
    ctx.track_step(image, hs, state, True, outputs="keypoints")   # a crop per slot
    graphs = {"track": capture(ctx, lambda: ctx.track_step(image, hs, state, False, outputs="keypoints"), state),
              "detect": capture(ctx, lambda: ctx.track_step(image, hs, state, True, outputs="keypoints"), state)}
    forces = {}
    for k in KS:
        f = torch.zeros(B, dtype=torch.int32, device="cuda")
        f[:k] = 1
        forces[k] = f
        graphs["slots_k%d" % k] = capture(ctx, lambda f=f: ctx.track_step_slots(image, hs, state, force=f, outputs="keypoints"), state)
    rounds = {n: [] for n in graphs}
    for _ in range(3):
        for n, g in graphs.items():
            rounds[n].append(time_replays(g, replays))
    us = {n: float(np.median(v)) for n, v in rounds.items()}
    out = {"track_step_us": round(us["track"], 1), "detect_step_us": round(us["detect"], 1), "slots": {}}
    for k in KS:
        pred = us["track"] + k / B * (us["detect"] - us["track"])
        out["slots"]["k%d" % k] = {"measured_us": round(us["slots_k%d" % k], 1), "predicted_us": round(pred, 1)}
    del graphs
    ctx.release_graphs()
    return out


def frames_per_s(ctx, B, host, n_steps, **kw):
    runner = FrameRunner(ctx, B, host[0].shape[1:3], **kw)
    redetected = []
    try:
        for _ in runner.stream(host[i % 2] for i in range(3)):   # warm-up: steps 0-2 (step 0 detects)
            pass
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        n = 0
        for r in runner.stream(host[i % 2] for i in range(n_steps)):
            n += 1
            if "track_detected" in r:
                redetected.append(int(r["track_detected"].sum()))
        dt = time.perf_counter() - t0
    finally:
        del runner
        ctx.release_graphs()
        gc.collect()
        torch.cuda.empty_cache()
    out = {"frames_per_s": round(B * n / dt, 1)}
    if redetected:
        out["slots_redetected_per_step"] = round(float(np.mean(redetected[1:] or redetected)), 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--replays", type=int, default=100)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--precisions", default="bf16x3,fp16")
    ap.add_argument("--no-frames", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_track_slots.py needs a CUDA device")
    ctx = runtime.Context(0)
    ctx.load_weights(Wt.synthetic_weights(0))
    res = {"card": card(), "results": {}}
    print(json.dumps(res["card"]), flush=True)
    B = args.batch
    for prec in args.precisions.split(","):
        ctx.set_precision(prec)
        r = res["results"][prec] = {"steps_b%d_240x320" % B: steps(ctx, B, args.replays)}
        print(prec, json.dumps(r), flush=True)
        if args.no_frames:
            continue
        H, W = 1080, 1920
        host = [np.stack([np.random.default_rng(100 * i + b).integers(0, 256, (H, W, 3), dtype=np.uint8) for b in range(B)])
                for i in range(2)]
        row = r["frame_runner_1080p_b%d" % B] = {
            "batch_redetect_1": frames_per_s(ctx, B, host, args.steps, track=True, redetect_every=1),
            "batch_redetect_None": frames_per_s(ctx, B, host, args.steps, track=True),
            "slots_redetect_%d" % B: frames_per_s(ctx, B, host, args.steps, track=True, detect="slots", redetect_every=B),
            "slots_redetect_None": frames_per_s(ctx, B, host, args.steps, track=True, detect="slots"),
        }
        print(prec, json.dumps(row), flush=True)
    print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

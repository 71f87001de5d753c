"""Cost of drawing on the device (h3d_draw_segments, FrameRunner(draw=True)).

    python scripts/bench_draw.py [--launches 200] [--steps 30] [--out result.json]

Kernel time: CUDA events over --launches launches into the same images, at B = 1 and 32 for 240x320, 1080x1920 and 2160x3840
frames, for a hand skeleton about a third of the frame high (20 segments, FrameRunner's default line width max(1, H / 240)) and for
a worst case of 24 segments spanning the frame.  Next to each time: box_MB, the bytes of the union boxes the CTAs walk, and
drawn_MB, the bytes of the pixels the call changes (read and written once each).
FrameRunner at 1080p, B = 32, bf16x3: the graph replay time (CUDA events over --steps replays) and stream()'s frames/s with host
frames, with draw off and on, alternated in one process, three runs each; stream() with draw on is also timed with drawn_every=0
(no drawn frame read back).  The drawing's share of the replay: after the replays, the step's own segments (the crop square and the
skeleton the graph drew) are rebuilt eagerly from its results, and CUDA events time, over --launches repetitions each, the kernel
on them (draw_ms) and the torch ops that build them (segments_ms).  The card's name and power limit are read in the same run.
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

from hand3d_b200 import runtime, weights as Wt          # noqa: E402
from hand3d_b200 import draw as D                       # noqa: E402
from hand3d_b200.frames import FrameRunner              # noqa: E402


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip().splitlines()[0]
    except Exception as e:      # the number is still reported, with the reason the power limit is missing
        info["power_limit_and_max_sm_clock"] = "unavailable (%s)" % e
    return info


def segments(kind, B, H, W, rng):
    if kind == "hand":
        size = np.float32([H, W]) / 3
        base = rng.uniform(0.1, 0.6, (B, 1, 2)).astype(np.float32) * np.float32([H, W])
        hw = torch.from_numpy(base + rng.uniform(0, 1, (B, 21, 2)).astype(np.float32) * size).cuda()
        return D.hand_segments(hw).contiguous(), D.PALETTE, max(1.0, H / 240.0)
    seg = (rng.uniform(0, 1, (B, 24, 4)) * np.float32([H, W, H, W])).astype(np.float32)
    return torch.from_numpy(seg).cuda(), rng.uniform(0, 255, (24, 3)).astype(np.float32), 1.0


def kernel_rows(ctx, launches):
    rows = []
    rng = np.random.default_rng(0)
    for H, W in ((240, 320), (1080, 1920), (2160, 3840)):
        for B in (1, 32):
            imgs = torch.randint(0, 256, (B, H, W, 3), dtype=torch.uint8, device="cuda")
            for kind in ("hand", "span"):
                seg, cols, lw = segments(kind, B, H, W, rng)
                before = imgs.clone()
                ctx.draw_segments(imgs, seg, cols, lw)
                drawn = int((imgs != before).any(-1).sum()) * 3 * 2
                s = seg.cpu().numpy()
                g = lw / 2 + 1.5
                lo_r = np.clip(np.minimum(s[..., 0], s[..., 2]).min(1) - g, 0, H - 1)
                hi_r = np.clip(np.maximum(s[..., 0], s[..., 2]).max(1) + g, 0, H - 1)
                lo_c = np.clip(np.minimum(s[..., 1], s[..., 3]).min(1) - g, 0, W - 1)
                hi_c = np.clip(np.maximum(s[..., 1], s[..., 3]).max(1) + g, 0, W - 1)
                box = int(((hi_r - lo_r + 1) * (hi_c - lo_c + 1)).sum()) * 3
                for _ in range(10):
                    ctx.draw_segments(imgs, seg, cols, lw)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                for _ in range(launches):
                    ctx.draw_segments(imgs, seg, cols, lw)
                e1.record()
                torch.cuda.synchronize()
                us = e0.elapsed_time(e1) * 1e3 / launches
                row = {"frame": "%dx%d" % (H, W), "B": B, "kind": kind, "segments": int(seg.shape[1]), "linewidth": lw,
                       "us_per_launch": round(us, 2), "box_MB": round(box / 1e6, 3), "drawn_MB": round(drawn / 1e6, 3),
                       "frame_MB": round(B * H * W * 3 / 1e6, 1)}
                print(json.dumps(row), flush=True)
                rows.append(row)
            del imgs
            torch.cuda.empty_cache()
    return rows


def replay_ms(runner, steps):
    for k in range(2):
        runner._graphs[k][0].replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for i in range(steps):
        runner._graphs[i & 1][0].replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def stream_fps(runner, batches, steps):
    items = [batches[i % len(batches)] for i in range(steps)]
    list(runner.stream(items[:4]))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in runner.stream(items):
        pass
    return steps * runner.B / (time.perf_counter() - t0)


def stream_fps_undrawn(runner, batches, steps):
    items = [batches[i % len(batches)] for i in range(steps)]
    list(runner.stream(items[:4], drawn_every=0))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in runner.stream(items, drawn_every=0):
        pass
    return steps * runner.B / (time.perf_counter() - t0)


def events_ms(fn, n):
    for _ in range(5):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def draw_share(ctx, runner, batch, launches):
    """The kernel and the segment-building ops of one drawing step, on the segments of a real step of `runner`."""
    frames = torch.from_numpy(batch).cuda()
    r = runner.submit(frames)
    torch.cuda.synchronize()
    center, scale, kp = r["center"].clone(), r["scale_crop"].clone(), r["keypoints_frame"].clone()

    def segments_of_step():
        return torch.cat([D.crop_box_segments(center, scale, runner.frame_hw, runner.size),
                          D.hand_segments(kp.to(torch.float32))], 1).contiguous()
    seg = segments_of_step()
    imgs = frames.clone()
    draw = events_ms(lambda: ctx.draw_segments(imgs, seg, runner._draw_colors, runner.draw_linewidth), launches)
    prep = events_ms(segments_of_step, launches)
    s = seg.cpu().numpy()
    H, W = runner.frame_hw
    g = runner.draw_linewidth / 2 + 1.5
    rows = np.clip(np.maximum(s[..., 0], s[..., 2]).max(1) + g, 0, H - 1) - np.clip(np.minimum(s[..., 0], s[..., 2]).min(1) - g, 0, H - 1) + 1
    cols = np.clip(np.maximum(s[..., 1], s[..., 3]).max(1) + g, 0, W - 1) - np.clip(np.minimum(s[..., 1], s[..., 3]).min(1) - g, 0, W - 1) + 1
    return {"draw_ms": round(draw, 3), "segments_ms": round(prep, 3), "box_fraction_of_frames": round(float((rows * cols).sum() / (len(s) * H * W)), 3)}


def frame_runner_rows(ctx, steps, launches, runs=3):
    B, hw = 32, (1080, 1920)
    ctx.set_precision("bf16x3")
    rng = np.random.default_rng(1)
    batches = [rng.integers(0, 256, (B,) + hw + (3,), dtype=np.uint8) for _ in range(2)]
    runners = {False: FrameRunner(ctx, B, hw), True: FrameRunner(ctx, B, hw, draw=True)}
    out = {False: {"replay_ms": [], "stream_fps": []}, True: {"replay_ms": [], "stream_fps": [], "stream_fps_drawn_every_0": []}}
    for _ in range(runs):
        for draw in (False, True):
            out[draw]["replay_ms"].append(round(replay_ms(runners[draw], steps), 3))
        for draw in (False, True):
            out[draw]["stream_fps"].append(round(stream_fps(runners[draw], batches, steps), 1))
        out[True]["stream_fps_drawn_every_0"].append(round(stream_fps_undrawn(runners[True], batches, steps), 1))
    res = {"frame": "1080x1920", "B": B, "precision": "bf16x3", "draw_off": out[False], "draw_on": out[True]}
    res["share"] = draw_share(ctx, runners[True], batches[0], launches)
    off, on = np.median(out[False]["replay_ms"]), np.median(out[True]["replay_ms"])
    res["replay_added_percent"] = round(100.0 * (on - off) / off, 2)
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_draw.py measures on the GPU; no CUDA device is present")
    res = {"card": card()}
    print(json.dumps(res["card"]), flush=True)
    ctx = runtime.default_context()
    ctx.load_weights(Wt.synthetic_weights(0))
    res["kernel"] = kernel_rows(ctx, args.launches)
    res["frame_runner"] = frame_runner_rows(ctx, args.steps, args.launches)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

"""A camera rig: one FrameRunner over cameras of different sizes and formats against one single-camera FrameRunner per camera.

    python scripts/bench_frames_rig.py [--steps 50] [--runs 5] [--launches 200] [--draw] [--out result.json]

Cameras: 1080x1920 NV12, 720x1280 YUYV and 480x640 RGB (--cameras repeats that set, e.g. --cameras 2 for six cameras).
1. Per-step time: CUDA events around --steps steps of device-resident frames (each step = one submit of the rig runner, or one submit
   of each single-camera runner), the median of --runs runs, rig and singles alternating.
2. The rig resize (h3d_resize_frames_rig: one kernel per format) against the sum of the single-size resizes of the same frames
   (h3d_resize_frames_fmt, B = 1 each): CUDA events over --launches launches, the best of --runs passes.
3. Kernels per step: the CUDA kernels torch.profiler records in one step of each (graph replays included).
The card's name, power limit and max SM clock are read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench_frames import card  # noqa: E402
from hand3d_b200 import frames as FR  # noqa: E402
from hand3d_b200 import runtime  # noqa: E402
from hand3d_b200 import weights as Wt  # noqa: E402

CAMERAS = [("nv12", (1080, 1920)), ("yuyv", (720, 1280)), ("rgb", (480, 640))]


def _events_ms(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def _kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type.name == "CUDA" and not e.name.startswith(("Memcpy", "Memset")))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--cameras", type=int, default=1, help="how many times the three cameras repeat")
    ap.add_argument("--draw", action="store_true", help="draw into the frames in the step")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_frames_rig.py needs a CUDA device")
    ctx = runtime.Context(0)
    ctx.load_weights(Wt.synthetic_weights(0))
    cams = CAMERAS * args.cameras
    fmts, hws = [c[0] for c in cams], [c[1] for c in cams]
    B = len(cams)
    g = torch.Generator(device="cuda").manual_seed(3)
    frames = [torch.randint(0, 256, FR.frame_shape(f, *hw), dtype=torch.uint8, device="cuda", generator=g) for f, hw in cams]
    res = {"card": card(), "cameras": ["%s %dx%d" % (f, *hw) for f, hw in cams], "draw": args.draw}
    print(json.dumps(res["card"]), flush=True)

    # 2. the resize alone
    out = torch.empty((B, 240, 320, 3), dtype=torch.float32, device="cuda")
    rig = lambda: ctx.resize_frames_rig(frames, 240, 320, True, out=out, pixel_formats=fmts)   # noqa: E731

    def singles():
        for b, (f, fr) in enumerate(zip(fmts, frames)):
            ctx.resize_frames(fr.unsqueeze(0), 240, 320, True, out=out[b:b + 1], pixel_format=f)
    for fn in (rig, singles):
        _events_ms(fn, 20)
    best_rig, best_sum = float("inf"), float("inf")
    for _ in range(args.runs):
        best_rig = min(best_rig, _events_ms(rig, args.launches))
        best_sum = min(best_sum, _events_ms(singles, args.launches))
    res["resize_us"] = {"rig": round(best_rig * 1000.0, 2), "sum_of_single_size": round(best_sum * 1000.0, 2),
                        "rig_over_sum": round(best_rig / best_sum, 3)}
    print(json.dumps(res["resize_us"]), flush=True)

    # 1. and 3. the whole step
    rig_runner = FR.FrameRunner(ctx, B, hws, pixel_format=fmts, draw=args.draw)
    one = [FR.FrameRunner(ctx, 1, hw, pixel_format=f, draw=args.draw) for f, hw in cams]
    step_rig = lambda: rig_runner.submit(frames)   # noqa: E731

    def step_singles():
        for r, fr in zip(one, frames):
            r.submit(fr.unsqueeze(0))
    for fn in (step_rig, step_singles):
        _events_ms(fn, 10)
    t_rig, t_one = [], []
    for _ in range(args.runs):
        t_rig.append(_events_ms(step_rig, args.steps))
        t_one.append(_events_ms(step_singles, args.steps))
    m_rig, m_one = statistics.median(t_rig), statistics.median(t_one)
    res["step_ms"] = {"rig": round(m_rig, 3), "single_camera_runners": round(m_one, 3), "speedup": round(m_one / m_rig, 2),
                      "rig_runs": [round(v, 3) for v in t_rig], "single_runs": [round(v, 3) for v in t_one]}
    print(json.dumps(res["step_ms"]), flush=True)
    res["kernels_per_step"] = {"rig": _kernels(step_rig), "single_camera_runners": _kernels(step_singles)}
    print(json.dumps(res["kernels_per_step"]), flush=True)
    # the rig's results equal the single-camera runners' (the check that makes the times comparable)
    a, b = rig_runner.submit(frames), [r.submit(fr.unsqueeze(0)) for r, fr in zip(one, frames)]
    torch.cuda.synchronize()
    res["keypoints_equal"] = bool(all(torch.equal(a["keypoints_frame"][i:i + 1], b[i]["keypoints_frame"]) for i in range(B)))
    del rig_runner, one
    ctx.release_graphs()
    print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

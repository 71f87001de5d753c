"""Images above 512 px a side: times the thread-block-cluster mask grower alone and the whole pipeline as a replayed CUDA graph.

    python scripts/bench_native.py [--steps 10] [--launches 200] [--out result.json]

Sizes 480x640, 720x1280, 1080x1920 and 2048x2048, batch sizes 1 and 8, bf16x3, synthetic weights.
1. The mask post-processing alone (h3d_seg_postprocess: the soft-max / arg-max kernel, then the grower) on fixed logits of two kinds:
   realistic blobs, whose growth reaches its fixed point after a few passes, and a serpentine corridor that runs every one of the
   max(H, W) // 10 passes.  CUDA events over --launches calls after warm-up; a separate torch.profiler run of the same calls gives the
   grower kernel's own time.
2. The pipeline (inference with the 3-D lifting, outputs="keypoints") on synthetic blob images, captured once per shape and replayed:
   CUDA events over --steps replays for the step time and images/s, a separate profiled replay for the grower's share of the step,
   and HandSegNet alone (eager, with its x8 up-sampling) for its images/s.
The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import grow_oracle as G  # noqa: E402
from hand3d_b200 import runtime  # noqa: E402
from hand3d_b200 import weights as Wt  # noqa: E402

SIZES = [(480, 640), (720, 1280), (1080, 1920), (2048, 2048)]
BATCHES = [1, 8]


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip().splitlines()[0]
    except Exception as e:      # the number is still reported, with the reason the power limit is missing
        info["power_limit_and_max_sm_clock"] = "unavailable (%s)" % e
    return info


def events_ms(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def kernel_us(fn, n):
    """{kernel name: total device µs per call} from a profiled run of n calls."""
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            out[e.name] = out.get(e.name, 0.0) + e.device_time_total / n
    return out


def grow_share(ks):
    return sum(v for k, v in ks.items() if "mask_grow" in k)


def bench_grower(ctx, B, H, W, kind, launches):
    logits = torch.from_numpy(G.logits_of([G.make_case(H, W, kind, seed=b) for b in range(B)])).cuda()
    call = lambda: ctx.seg_postprocess(logits)   # noqa: E731
    for _ in range(5):
        call()
    torch.cuda.synchronize()
    ms = events_ms(call, launches)
    ks = kernel_us(call, min(launches, 20))
    return {"size": "%dx%d" % (H, W), "B": B, "logits": kind, "passes_max": max(H, W) // 10,
            "seg_postprocess_us": round(ms * 1000.0, 1), "grow_kernel_us": round(grow_share(ks), 1)}


def bench_pipeline(ctx, B, H, W, steps):
    img = torch.from_numpy(Wt.synthetic_blob_images(B, H, W, seed=3)).cuda()
    hs = torch.from_numpy(Wt.synthetic_hand_side(B, seed=4)).cuda()
    replay, _ = ctx.capture_pipeline(img, hs, True, outputs="keypoints")
    for _ in range(3):
        replay()
    torch.cuda.synchronize()
    ms = events_ms(replay, steps)
    ks = kernel_us(replay, 2)
    del replay
    ctx.release_graphs()
    grow = grow_share(ks)
    seg = lambda: ctx.handsegnet(img)   # noqa: E731   HandSegNet alone, with its x8 up-sampling
    seg()
    torch.cuda.synchronize()
    seg_ms = events_ms(seg, max(2, steps // 2))
    return {"size": "%dx%d" % (H, W), "B": B, "step_ms": round(ms, 3), "images_per_s": round(B * 1000.0 / ms, 1),
            "grow_us": round(grow, 1), "grow_share_of_step": round(grow / (ms * 1000.0), 4),
            "handsegnet_eager_ms": round(seg_ms, 3), "handsegnet_images_per_s": round(B * 1000.0 / seg_ms, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_native.py needs a CUDA device")
    ctx = runtime.Context(0)
    ctx.load_weights(Wt.synthetic_weights(0, seg_shift=0.15))
    ctx.set_precision("bf16x3")
    ctx.ensure_workspace(max(BATCHES), 2048, 2048)   # once: captured graphs need a workspace that no longer grows
    res = {"card": card(), "grower": [], "pipeline": []}
    for H, W in SIZES:
        for B in BATCHES:
            for kind in ("blobs", "serpentine"):
                res["grower"].append(bench_grower(ctx, B, H, W, kind, args.launches))
                print(json.dumps(res["grower"][-1]), flush=True)
    for H, W in SIZES:
        for B in BATCHES:
            res["pipeline"].append(bench_pipeline(ctx, B, H, W, args.steps))
            print(json.dumps(res["pipeline"][-1]), flush=True)
    print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

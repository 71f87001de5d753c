"""Per-layer time of the tensor-core convolution (conv_tc_kernel) in the config-4 step.

Runs the full pipeline (32 images of 320x320, bf16x3 by default) under torch.profiler with CUDA activities.  The conv_tc_kernel
launches of a step are matched, in launch order, with the layer table of hand3d_b200/arch.py; per layer the script reports the
median kernel time, the algorithmic and executed TFLOP/s, and the L2 -> shared-memory bytes the TMA boxes move (modelled from the
tile geometry: every A and B box the kernel loads) with the resulting TB/s.

    python scripts/profile_conv_layers.py --out DIR      # needs the GPU; writes DIR/profile_conv_layers.json
    python scripts/profile_conv_layers.py --model-only   # the modelled bytes / FLOPs per layer, no GPU
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from hand3d_b200 import arch  # noqa: E402

BM, BK = 128, 64
TILE_CANDIDATES = [(16, 8, 1), (8, 16, 1), (32, 4, 1), (4, 32, 1), (64, 2, 1), (128, 1, 1), (8, 8, 2), (16, 4, 2), (4, 16, 2),
                   (8, 4, 4), (4, 8, 4), (4, 4, 8), (8, 2, 8), (2, 2, 32), (1, 1, 128)]   # csrc/conv_wgmma.cu: choose_tile
PASSES = {"bf16x3": 3, "fp16x3": 3, "fp16": 1, "bf16": 1}   # fp16_f8c runs the lifting stage on CUDA cores


def cdiv(a, b):
    return -(-a // b)


def choose_tile(B, H, W, pool):
    best = None
    for tw, th, tb in TILE_CANDIDATES:
        if pool and not (tw % 2 == 0 and tw <= 16 and th % 2 == 0):
            continue
        n = cdiv(W, tw) * cdiv(H, th) * cdiv(B, tb)
        if best is None or n < best[0]:
            best = (n, (tw, th, tb))
    return best[1]


def tc_layers(B=32, H=320, W=320, crop=256):
    """The conv_tc_kernel launches of one full-pipeline step in launch order: (name, B, H, W, k, Cin, Cout, Cin_pad, pool, passes)
    with H, W the layer's input size (the kernel computes the stride-1 result; pool 1 = fused 2x2 max-pool, 2 = stride 2)."""
    out = []
    for scope, layers, h, w in (("HandSegNet", arch.HANDSEGNET, H, W), ("PoseNet2D", arch.POSENET2D, crop, crop)):
        for name, k, s, cin, cout, _ in layers:
            if name == "conv1_1":
                continue
            pool = 1 if name in arch.HANDSEGNET_POOL_AFTER else 0
            cin_pad = 192 if name in ("conv6_1", "conv7_1") and scope == "PoseNet2D" else 64 * cdiv(cin, 64)
            out.append(("%s/%s" % (scope, name), B, h, w, k, cin, cout, cin_pad, pool, None))
            if pool:
                h, w = h // 2, w // 2
    # the lifting stage always runs 3-pass; ViewpointNet's pyramid is enqueued first (side stream), then PosePrior's
    for scope, layers in (("ViewpointNet", arch.VIEWPOINT), ("PosePrior", arch.POSEPRIOR)):
        h = w = 32
        for name, k, s, cin, cout, _ in layers:
            if k == 0:
                continue
            out.append(("%s/%s" % (scope, name), B, h, w, k, cin, cout, 64 * cdiv(cin, 64), 2 if s == 2 else 0, 3))
            h, w = h // s, w // s
    return out


def layer_model(layer, precision):
    """Tiles and modelled traffic of one layer (the rules of tc_conv_plan_create)."""
    name, B, H, W, k, cin, cout, cin_pad, pool, passes = layer
    passes = passes or PASSES[precision]
    cout_pad = 64 * cdiv(cout, 64)
    bn = 128 if cout_pad % 128 == 0 else 64
    if H * W <= 256 or passes == 4:
        bn = 64
    tw, th, tb = choose_tile(B, H, W, pool == 1)
    m_tiles = cdiv(W, tw) * cdiv(H, th) * cdiv(B, tb)
    n_tiles = cout_pad // bn
    kblocks = k * k * cin_pad // BK
    planes = 1 if passes == 1 else 2
    a_bytes, b_bytes = planes * BM * BK * 2, planes * bn * BK * 2      # per K block
    ho, wo = (H // 2, W // 2) if pool == 2 else (H, W)
    return {
        "layer": name, "B": B, "H": H, "W": W, "k": k, "cin": cin, "cout": cout, "pool": pool, "passes": passes, "BN": bn,
        "tile": [tw, th, tb], "m_tiles": m_tiles, "n_tiles": n_tiles,
        "flop_alg": 2 * B * ho * wo * k * k * cin * cout,
        "flop_exec": 2 * m_tiles * BM * n_tiles * bn * kblocks * BK * (1 if passes == 1 else 3),
        "l2_smem_bytes": m_tiles * n_tiles * kblocks * (a_bytes + b_bytes),
    }


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"name": name, "power_limit": power, "clocks_max_sm": clock}


def conv_kernel_times(trace_path):
    """conv_tc_kernel durations (us) in host launch order (correlation id): the side-stream pyramid may overlap on the device."""
    with open(trace_path) as f:
        ev = json.load(f)["traceEvents"]
    ks = [e for e in ev if e.get("cat") == "kernel" and "conv_tc_kernel" in e.get("name", "")]
    ks.sort(key=lambda e: e["args"]["correlation"])
    return [(e["name"], float(e["dur"])) for e in ks]


def profile(args):
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile

    from hand3d_b200 import runtime, weights as Wt

    if not torch.cuda.is_available():
        raise SystemExit("profile_conv_layers.py: no CUDA device (use --model-only for the modelled numbers)")
    info = gpu_info()
    B, H, W = 32, 320, 320
    ctx = runtime.Context(0, precision=args.precision)
    ctx.load_weights(Wt.synthetic_weights(0))
    ctx.ensure_workspace(B, H, W)
    img = torch.from_numpy(Wt.synthetic_images(B, H, W, seed=1000)).cuda()
    hs = torch.from_numpy(Wt.synthetic_hand_side(B, seed=2000)).cuda()
    layers = tc_layers(B, H, W)
    times = [[] for _ in layers]
    with tempfile.TemporaryDirectory() as td:
        for _ in range(args.warmup):
            ctx.pipeline(img, hs, True, outputs="keypoints")
        torch.cuda.synchronize()
        for rep in range(args.reps):
            with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.steps):
                    ctx.pipeline(img, hs, True, outputs="keypoints")
                torch.cuda.synchronize()
            path = os.path.join(td, "trace_%d.json" % rep)
            prof.export_chrome_trace(path)
            ks = conv_kernel_times(path)
            if len(ks) != args.steps * len(layers):
                raise SystemExit("expected %d conv_tc_kernel launches per step, found %d in %d steps" % (len(layers), len(ks), args.steps))
            for i, (kname, dur) in enumerate(ks):
                li = i % len(layers)
                bn = layer_model(layers[li], args.precision)["BN"]
                if "conv_tc_kernel<%d," % bn not in kname:
                    raise SystemExit("launch %d (%s) does not match layer %s (BN %d)" % (i, kname, layers[li][0], bn))
                times[li].append(dur)
    ctx.check_errors()
    rows = []
    for li, layer in enumerate(layers):
        m = layer_model(layer, args.precision)
        us = statistics.median(times[li])
        m.update({"us": us, "us_min": min(times[li]), "us_max": max(times[li]), "tflops_alg": m["flop_alg"] / us * 1e-6,
                  "tflops_exec": m["flop_exec"] / us * 1e-6, "l2_smem_tb_s": m["l2_smem_bytes"] / us * 1e-6})
        rows.append(m)
    tot = {"us": sum(r["us"] for r in rows), "l2_smem_bytes": sum(r["l2_smem_bytes"] for r in rows),
           "flop_alg": sum(r["flop_alg"] for r in rows), "flop_exec": sum(r["flop_exec"] for r in rows)}
    result = {"gpu": info, "workload": "config 4 step: full pipeline, %d images of %dx%d, %s" % (B, H, W, args.precision),
              "reps": args.reps, "steps_per_rep": args.steps, "layers": rows, "total": tot}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "profile_conv_layers.json"), "w") as f:
        json.dump(result, f, indent=1)
    print("%s, power limit %s, max SM clock %s" % (info["name"], info["power_limit"], info["clocks_max_sm"]))
    print("%-26s %4s %6s | %9s %7s %7s | %7s %6s" % ("layer", "BN", "tiles", "us", "TF alg", "TF exe", "GB", "TB/s"))
    for r in rows:
        print("%-26s %4d %6d | %9.1f %7.0f %7.0f | %7.2f %6.2f" % (r["layer"], r["BN"], r["m_tiles"] * r["n_tiles"], r["us"], r["tflops_alg"],
                                                                  r["tflops_exec"], r["l2_smem_bytes"] / 1e9, r["l2_smem_tb_s"]))
    print("total conv_tc_kernel: %.0f us per step, %.0f TFLOP/s algorithmic, %.0f executed, modelled L2->SMEM %.1f GB = %.2f TB/s" % (
        tot["us"], tot["flop_alg"] / tot["us"] * 1e-6, tot["flop_exec"] / tot["us"] * 1e-6, tot["l2_smem_bytes"] / 1e9,
        tot["l2_smem_bytes"] / tot["us"] * 1e-6))


def model_only(args):
    tot = 0
    print("%-26s %4s %6s %9s %8s" % ("layer", "BN", "tiles", "tile", "GB"))
    for layer in tc_layers():
        m = layer_model(layer, args.precision)
        tot += m["l2_smem_bytes"]
        print("%-26s %4d %6d %9s %8.2f" % (m["layer"], m["BN"], m["m_tiles"] * m["n_tiles"], "x".join(map(str, m["tile"])), m["l2_smem_bytes"] / 1e9))
    print("total modelled L2->SMEM per step: %.1f GB" % (tot / 1e9))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", default="profile_out", help="output directory for profile_conv_layers.json")
    ap.add_argument("--precision", default="bf16x3", choices=sorted(PASSES))
    ap.add_argument("--reps", type=int, default=3, help="profiled runs")
    ap.add_argument("--steps", type=int, default=3, help="profiled steps per run")
    ap.add_argument("--warmup", type=int, default=3, help="untimed steps before the first run")
    ap.add_argument("--model-only", action="store_true", help="print the modelled bytes per layer and exit (no GPU)")
    args = ap.parse_args()
    if args.model_only:
        model_only(args)
    else:
        profile(args)


if __name__ == "__main__":
    main()

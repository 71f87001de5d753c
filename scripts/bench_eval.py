"""Evaluation loops: samples/s of the four evaluation scripts' loops three ways, and h3d_eval_stats alone.

    python scripts/bench_eval.py [--reps 2] [--out result.json]

1. Each demo loop (examples/eval2d_demo.py, eval2d_gt_cropped_demo.py, eval3d_demo.py, eval_full_demo.py) over synthetic records, RHD
   at 2728 records and STB at 1024, at B = 16 and 32; eval3d with the lifting stage as `direct` and `proposed` (eval_full runs
   ColorHandPose3DNetwork, whose lifting is `proposed`):
   (a) the host reader, eager inference and EvalUtil (the demos' default);
   (b) the resident reader, eager inference and DeviceEvalUtil (--device-resident);
   (c) the resident reader with one CUDA graph per batch (--device-resident --graph).
   A pass is ceil(n / B) batches and get_measures, timed by the host clock (get_measures ends in a synchronise), after a warm-up of
   three batches (which also captures the graph of (c)).  The modes alternate within each repetition.
2. h3d_eval_stats alone, K = 21, T = 20 and 100, N = 2728, 41 258 and 10^6 samples of each dtype: CUDA events over 20 launches.
The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from examples._synthetic_db import fake_rhd, fake_stb  # noqa: E402
from hand3d_b200 import runtime  # noqa: E402
from hand3d_b200.data.BinaryDbReader import BinaryDbReader, BinaryDbReaderSTB  # noqa: E402
from hand3d_b200.train_loop import GraphedIteration  # noqa: E402
from hand3d_b200.utils.general import DeviceEvalUtil, EvalUtil  # noqa: E402
from hand3d_b200.weights import synthetic_weights  # noqa: E402


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip().splitlines()[0]
    except Exception as e:      # the number is still reported, with the reason the power limit is missing
        info["power_limit_and_max_sm_clock"] = "unavailable (%s)" % e
    return info


def _demo(name):
    import importlib
    return importlib.import_module("examples." + name)


def _setup(script, variant, path, B, resident):
    """(reader, step) of one demo loop, as the demo builds them."""
    ctx = runtime.default_context()
    w = synthetic_weights(0)
    if script == "eval3d":
        from hand3d_b200.nets.PosePriorNetwork import PosePriorNetwork
        net = PosePriorNetwork(variant)
        net.init(None, weights={k: v for k, v in w.items() if k.startswith(("PosePrior", "ViewpointNet"))})
        reader = BinaryDbReader(mode='evaluation', shuffle=False, hand_crop=True, use_wrist_coord=False, batch_size=B, path_to_db=path,
                                device_resident=resident)
        return reader, _demo("eval3d_demo").make_step(net)
    from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork
    net = ColorHandPose3DNetwork()
    if script == "eval_full":
        net.init(None, weights=w)
        reader = BinaryDbReaderSTB(mode='evaluation', shuffle=False, use_wrist_coord=False, batch_size=B, path_to_db=path,
                                   device_resident=resident)
        return reader, _demo("eval_full_demo").make_step(net, ctx)
    net.init(None, weights=w, exclude_var_list=['PosePrior', 'ViewpointNet'])
    if script == "eval2d":
        reader = BinaryDbReader(mode='evaluation', shuffle=False, use_wrist_coord=True, scale_to_size=True, batch_size=B, path_to_db=path,
                                device_resident=resident)
        return reader, _demo("eval2d_demo").make_step(net, resident)
    reader = BinaryDbReader(mode='evaluation', shuffle=False, hand_crop=True, use_wrist_coord=False, batch_size=B, path_to_db=path,
                            device_resident=resident)
    return reader, _demo("eval2d_gt_cropped_demo").make_step(net, ctx, resident)


def time_loop(script, variant, path, n, B, mode):
    resident = mode != "a"
    reader, step = _setup(script, variant, path, B, resident)
    util = DeviceEvalUtil(num_samples=n) if resident else EvalUtil()

    def iteration():
        step(reader.get(), util)

    run = GraphedIteration(iteration) if mode == "c" else iteration
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    if resident:
        util.reset()
    else:
        util.data = [list() for _ in range(util.num_kp)]
    t0 = time.perf_counter()
    for _ in range(0, n, B):
        run()
    util.get_measures(0.0, 0.05, 20)
    dt = time.perf_counter() - t0
    del run, reader, util
    torch.cuda.empty_cache()
    return n / dt


def time_stats(N, T, dtype, launches=20):
    ctx = runtime.default_context()
    g = torch.Generator(device="cuda").manual_seed(N)
    ev = DeviceEvalUtil(num_samples=N)
    gt = torch.rand((N, 21, 3), generator=g, device="cuda", dtype=dtype)
    pred = torch.rand((N, 21, 3), generator=g, device="cuda", dtype=dtype)
    ev.feed(gt, torch.ones((N, 21), dtype=torch.uint8, device="cuda"), pred)
    thr = torch.from_numpy(np.linspace(0.0, 1.5, T)).cuda()
    for _ in range(3):
        ctx.eval_stats(ev._store, 21, N, dtype, thr)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        ctx.eval_stats(ev._store, 21, N, dtype, thr)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000.0 / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = {"card": card(), "loops": [], "stats_us": []}
    tmp = tempfile.mkdtemp()
    paths = {"rhd": os.path.join(tmp, "rhd.bin"), "stb": os.path.join(tmp, "stb.bin")}
    sizes = {"rhd": 2728, "stb": 1024}
    with open(paths["rhd"], "wb") as f:
        f.write(fake_rhd(sizes["rhd"], seed=1))
    with open(paths["stb"], "wb") as f:
        f.write(fake_stb(sizes["stb"], seed=2))
    try:
        cases = [("eval2d", None, "rhd"), ("eval2d_gt_cropped", None, "rhd"), ("eval3d", "direct", "rhd"), ("eval3d", "proposed", "rhd"),
                 ("eval_full", "proposed", "stb")]
        for script, variant, kind in cases:
            for B in (16, 32):
                row = {"script": script, "lifting": variant, "B": B, "samples": sizes[kind]}
                for rep in range(args.reps):
                    for mode in ("a", "b", "c"):
                        row.setdefault(mode, []).append(round(time_loop(script, variant, paths[kind], sizes[kind], B, mode), 1))
                row["speedup_c_over_a"] = round(np.median(row["c"]) / np.median(row["a"]), 2)
                print(json.dumps(row), flush=True)
                res["loops"].append(row)
        for dtype in (torch.float32, torch.float64):
            for N in (2728, 41258, 10 ** 6):
                for T in (20, 100):
                    r = {"dtype": str(dtype).split(".")[-1], "N": N, "T": T, "us": round(time_stats(N, T, dtype), 1)}
                    print(json.dumps(r), flush=True)
                    res["stats_us"].append(r)
    finally:
        for p in paths.values():
            if os.path.exists(p):
                os.unlink(p)
        os.rmdir(tmp)
    print(json.dumps(res["card"]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

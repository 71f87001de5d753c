"""Cost of the pipeline's x8 up-sampling + key-point arg-max (h3d_upsample_detect_keypoints, resize_argmax_pow2_kernel).

    python scripts/bench_upsample_argmax.py [--launches 200] [--repeats 3] [--lib A.so --lib B.so ...] [--out result.json]

PoseNet's 21 score maps of 32 x 32 go to 256 x 256 (nets/ColorHandPose3DNetwork.py:96-97) at B = 1, 8 and 32 images.  Kernel time:
CUDA events around --launches back-to-back calls after a warm-up, divided by the launches (each call is the scratch memset, the
up-sampling kernel and the small decode kernel); MB is the bytes the call must move (the maps read once, the up-sampled maps written
once), GB/s those bytes over the time.  Each --lib (default: the in-tree library) is timed in a child process of its own, the libraries
alternating over --repeats rounds; the median of the rounds is reported.  Every child also hashes the outputs of the seeded inputs, and
the libraries must agree.  The card's name and power limit are read in the same run."""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
BATCHES = (1, 8, 32)


def card():
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        info["power_limit_and_max_sm_clock"] = q.stdout.strip().splitlines()[0]
    except Exception as e:      # the number is still reported, with the reason the power limit is missing
        info["power_limit_and_max_sm_clock"] = "unavailable (%s)" % e
    return info


def child(lib_path, launches):
    from hand3d_b200 import _lib
    if lib_path:
        _lib.LIB_PATH = os.path.abspath(lib_path)
    import numpy as np
    import torch
    from hand3d_b200 import runtime
    ctx = runtime.default_context()
    rows = []
    for B in BATCHES:
        x = torch.from_numpy(np.random.default_rng(B).normal(size=(B, 32, 32, 21)).astype(np.float32)).cuda()
        up = torch.empty((B, 256, 256, 21), device="cuda")
        uv = torch.empty((B, 21, 2), dtype=torch.int32, device="cuda")
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

        def call():
            _lib.check(ctx.lib.h3d_upsample_detect_keypoints(ctx.h, C.c_void_p(x.data_ptr()), B, 32, 32, 256, 256, C.c_void_p(up.data_ptr()),
                                                             C.c_void_p(uv.data_ptr()), st), "h3d_upsample_detect_keypoints")
        for _ in range(20):
            call()
        torch.cuda.synchronize()
        digest = hashlib.sha256(up.cpu().numpy().tobytes() + uv.cpu().numpy().tobytes()).hexdigest()[:16]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            call()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / launches
        mb = B * (32 * 32 + 256 * 256) * 21 * 4 / 1e6
        rows.append({"B": B, "ms": ms, "MB": mb, "GB_per_s": mb / ms, "outputs": digest})
    ctx.check_errors()
    print(json.dumps(rows))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--lib", action="append", default=None, help="a libhand3d_b200.so to time (repeatable; default: the in-tree one)")
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child is not None:
        child(args.child, args.launches)
        return
    libs = args.lib or [""]
    runs = {lib: [] for lib in libs}
    for _ in range(args.repeats):
        for lib in libs:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", lib, "--launches", str(args.launches)],
                               stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
            if r.returncode:
                raise SystemExit("child for %r failed:\n%s" % (lib or "in-tree", r.stdout[-4000:]))
            runs[lib].append(json.loads(r.stdout.strip().splitlines()[-1]))
    result = {"card": card(), "launches": args.launches, "repeats": args.repeats, "rows": []}
    for lib in libs:
        for i, B in enumerate(BATCHES):
            ms = sorted(rep[i]["ms"] for rep in runs[lib])
            first = runs[lib][0][i]
            result["rows"].append({"lib": lib or "in-tree", "B": B, "ms_median": ms[len(ms) // 2], "ms_all": ms, "MB": first["MB"],
                                   "GB_per_s": first["MB"] / ms[len(ms) // 2], "outputs": first["outputs"]})
    digests = {(row["B"], row["outputs"]) for row in result["rows"]}
    result["outputs_agree"] = len(digests) == len(BATCHES)
    print(json.dumps(result, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    if not result["outputs_agree"]:
        raise SystemExit("the libraries' outputs differ")


if __name__ == "__main__":
    main()

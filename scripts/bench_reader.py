#!/usr/bin/env python
"""Times BinaryDbReader.get() in the three training configurations of the reference's scripts (training_handsegnet.py:37-39,
training_posenet.py:37-39, training_lifting.py:44-46) at B = 8 and 32, and sets it beside one training step of the network each
script trains, measured in the same run.

Per configuration and batch size, medians over --iters calls after --warmup:
  get_ms       wall time of get() (synchronised), shuffle, gather, upload and every launch included;
  host_ms      the host part that moves bytes: gathering the records from the memory-mapped file, pinning and uploading them;
  device_ms    CUDA events around get() with the records already on the device (the stream span of the reader's kernels);
  kernels_ms   the reader's CUDA kernel time from torch.profiler (kernels only, no gaps);
  step_ms      one eager training step (forward, loss, backward, Adam; bf16x3) of HandSegNet / PoseNet2D on 256 x 256 inputs or of
               PosePrior + ViewpointNet ('proposed'), from scripts/bench_train_step.py / bench_train_lifting.py.
The records are synthetic (examples/_synthetic_db.py) in a temporary file; the timing does not depend on their content.

    python scripts/bench_reader.py [--batch 8 32] [--iters 20] [--out reader.json]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from hand3d_b200 import runtime, weights as Wt  # noqa: E402
from hand3d_b200.data.BinaryDbReader import BinaryDbReader  # noqa: E402
from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork  # noqa: E402
from examples._synthetic_db import fake_rhd  # noqa: E402
import bench_train_lifting as BL  # noqa: E402
import bench_train_step as BT  # noqa: E402

CONFIGS = {
    "handsegnet": dict(shuffle=True, hue_aug=True, random_crop_to_size=True),
    "posenet": dict(shuffle=True, use_wrist_coord=False, hand_crop=True, coord_uv_noise=True, crop_center_noise=True),
    "lifting": dict(shuffle=True, hand_crop=True, use_wrist_coord=False, coord_uv_noise=True, crop_center_noise=True, crop_offset_noise=True,
                    crop_scale_noise=True),
}


def median_ms(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def kernels_ms(fn, iters):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    return sum(e.self_device_time_total for e in prof.key_averages() if "memcpy" not in e.key.lower()) / 1e3 / iters


def bench_reader(path, name, B, warmup, iters):
    rd = BinaryDbReader(mode="training", batch_size=B, path_to_db=path, seed=1, **CONFIGS[name])
    r = {"config": name, "B": B, "get_ms": median_ms(rd.get, warmup, iters)}
    serials = list(range(B))
    r["host_ms"] = median_ms(lambda: rd._file.gather(serials), warmup, iters)
    records = rd._file.gather(serials)
    rd._file.gather = lambda s: records            # device part alone: the records stay on the device
    r["device_ms"] = BT.time_ms(lambda: rd._get(serials), warmup, iters)
    r["kernels_ms"] = kernels_ms(lambda: rd._get(serials), iters)
    return r


def step_ms(name, B, warmup, iters):
    if name == "lifting":
        step = BL.setup("proposed", B)[-1]
    else:
        ColorHandPose3DNetwork().init(weights=Wt.synthetic_weights(0))
        step = BT.setup("HandSegNet" if name == "handsegnet" else "PoseNet2D", B, 256)[-1]
    return median_ms(step, warmup, iters)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batch", type=int, nargs="*", default=[8, 32])
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    runtime.default_context().set_precision("bf16x3")
    res = []
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "rhd_training.bin")
        with open(path, "wb") as f:
            f.write(fake_rhd(64))
        for B in a.batch:
            for name in CONFIGS:
                r = bench_reader(path, name, B, a.warmup, a.iters)
                r["step_ms"] = step_ms(name, B, a.warmup, a.iters)
                r["get_share_of_get_plus_step"] = r["get_ms"] / (r["get_ms"] + r["step_ms"])
                print(json.dumps(r))
                sys.stdout.flush()
                res.append(r)
                torch.cuda.empty_cache()
    doc = {"gpu": BT.gpu_info(), "results": res}
    print(json.dumps(doc["gpu"]))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()

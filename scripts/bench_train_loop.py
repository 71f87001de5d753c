#!/usr/bin/env python
"""Times a whole training iteration, reading included, in the three configurations of the reference's training scripts
(training_handsegnet.py, training_posenet.py, training_lifting.py: their reader flags, shuffled, seeded) at B = 8 and 32, in three
modes:
  a  host_eager     BinaryDbReader.get() on the host path, then the eager step (today's demo loop);
  b  host_graph     host get(), its items copied into the static inputs of a step replayed from a CUDA graph;
  c  resident_graph BinaryDbReader(..., device_resident=True): get(), forward, loss, backward and Adam replayed from one CUDA graph.
A step is zero_grad, forward, loss, backward and the Adam update in bf16x3, as in examples/train_*_demo.py: HandSegNet on the 256 x 256
windows, PoseNet2D on the 256 x 256 crops, PosePrior + ViewpointNet ('proposed') on the 256 x 256 score maps.  Each figure is the
median wall time of --iters iterations after --warmup, each followed by a device synchronise inside the timed window.  The records
are synthetic (examples/_synthetic_db.py) in a temporary file; the timing does not depend on their content.

    python scripts/bench_train_loop.py [--batch 8 32] [--iters 50] [--out train_loop.json]
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

from hand3d_b200 import autograd as A, runtime, weights as Wt  # noqa: E402
from hand3d_b200.data.BinaryDbReader import BinaryDbReader  # noqa: E402
from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork  # noqa: E402
from hand3d_b200.nets.PosePriorNetwork import PosePriorNetwork  # noqa: E402
from hand3d_b200.optim import Adam  # noqa: E402
from hand3d_b200.train_loop import GraphedIteration  # noqa: E402
from examples._synthetic_db import fake_rhd  # noqa: E402
from bench_train_step import gpu_info  # noqa: E402

CONFIGS = {
    "handsegnet": dict(shuffle=True, hue_aug=True, random_crop_to_size=True),
    "posenet": dict(shuffle=True, use_wrist_coord=False, hand_crop=True, coord_uv_noise=True, crop_center_noise=True),
    "lifting": dict(shuffle=True, hand_crop=True, use_wrist_coord=False, coord_uv_noise=True, crop_center_noise=True, crop_offset_noise=True,
                    crop_scale_noise=True),
}
MODES = ("host_eager", "host_graph", "resident_graph")


def make_step(name):
    """step(data) -> loss (detached): one training step of the network `name` trains, on the reader's items."""
    ctx = runtime.default_context()
    if name == "lifting":
        ctx.load_weights(Wt.xavier_weights(0))
        net = PosePriorNetwork("proposed")
        params = [p for s in ("PosePrior", "ViewpointNet") for p in ctx.variables(s).values()]
    else:
        scope = "HandSegNet" if name == "handsegnet" else "PoseNet2D"
        net = ColorHandPose3DNetwork()
        net.init(weights={k: v for k, v in Wt.synthetic_weights(0).items() if k.startswith(scope + "/")})
        params = list(ctx.variables(scope).values())
    for p in params:
        p.grad = None
    opt = Adam(params, lr=1e-5)

    def step(d):
        if name == "handsegnet":
            loss = A.softmax_xent_loss(net.inference_detection(d["image"], train=True)[0], d["hand_mask"].float())
        elif name == "posenet":
            s = d["scoremap"].shape
            vis = d["keypoint_vis21"].reshape(s[0], s[3]).float()
            loss = sum(A.scoremap_loss(A.resize_bilinear(m, s[1], s[2]), d["scoremap"], vis)
                       for m in net.inference_pose2d(d["image_crop"], train=True))
        else:
            _, coord, R = net.inference(d["scoremap"], d["hand_side"], True, train=True)
            loss = A.mse_loss(coord, d["keypoint_xyz21_can"]) + A.mse_loss(R, d["rot_mat"])
        opt.zero_grad()
        loss.backward()
        opt.step()
        return loss.detach()

    return step


def make_iteration(mode, name, B, path):
    rd = BinaryDbReader(mode="training", batch_size=B, path_to_db=path, seed=1, device_resident=mode == "resident_graph",
                        **CONFIGS[name])
    step = make_step(name)
    if mode == "host_eager":
        return lambda: step(rd.get())
    if mode == "resident_graph":
        return GraphedIteration(lambda: step(rd.get()))
    static = {k: v.clone() for k, v in rd.get().items()}
    graphed = GraphedIteration(lambda: step(static))

    def iteration():
        for k, v in rd.get().items():
            static[k].copy_(v)
        return graphed()
    return iteration


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


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batch", type=int, nargs="*", default=[8, 32])
    ap.add_argument("--configs", nargs="*", default=list(CONFIGS), choices=list(CONFIGS))
    ap.add_argument("--warmup", type=int, default=5, help="untimed iterations (>= 3: two eager warm-ups and the capture)")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--records", type=int, default=256, help="records in the synthetic file")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.warmup < 3 or a.iters < 1:
        ap.error("--warmup must be >= 3 and --iters >= 1")
    torch.cuda.set_device(0)
    runtime.default_context().set_precision("bf16x3")
    res = []
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "rhd_training.bin")
        with open(path, "wb") as f:
            f.write(fake_rhd(a.records))
        for B in a.batch:
            for name in a.configs:
                r = {"config": name, "B": B}
                for mode in MODES:
                    it = make_iteration(mode, name, B, path)
                    try:
                        r[mode + "_ms"] = median_ms(it, a.warmup, a.iters)
                    except Exception:
                        # a trapped kernel poisons the context; the error word names a timed-out barrier wait (h3d_check_errors)
                        print("failed in %s, %s, B = %d" % (mode, name, B), file=sys.stderr)
                        runtime.default_context().check_errors()
                        raise
                    del it
                    torch.cuda.synchronize()
                    torch.cuda.empty_cache()
                r["speedup_c_over_a"] = r["host_eager_ms"] / r["resident_graph_ms"]
                print(json.dumps(r))
                sys.stdout.flush()
                res.append(r)
    doc = {"gpu": gpu_info(), "precision": "bf16x3", "iters": a.iters, "warmup": a.warmup, "results": res}
    print(json.dumps(doc["gpu"]))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()

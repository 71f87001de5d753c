"""Times one training step of PoseNet2D and of HandSegNet on the project's kernels, eager and replayed from a CUDA graph.

Shapes: PoseNet2D at B = 8 crops of 256x256 with its three score maps up-sampled to 256x256 and the score-map loss
(training_posenet.py:38-61); HandSegNet at B = 8 images of 256x256, the shape of the reference's random_crop_to_size, with the
softmax cross-entropy (training_handsegnet.py:37-60).  A step is zero_grad, forward, loss, backward and the Adam update
(hand3d_b200.optim.Adam).  Synthetic weights and inputs: the timings do not depend on the values.

Reported per network, all measured in the same run:
  * step_eager_ms, step_graph_ms: the whole step, eagerly and as one replayed CUDA graph (median of --iters CUDA-event timings
    after --warmup untimed runs);
  * net_fwd_bwd_ms: forward + backward of the network alone (convolutions, pools, concat; no resize, loss or Adam), replayed from a
    CUDA graph like the kernel groups below, so that it is GPU time as well;
  * resize_fwd_bwd_ms, loss_fwd_bwd_ms, adam_ms: GPU time of the training kernels (csrc/train.cu plus the resize forward) with the
    step's shapes: each group is captured --reps times back to back into one CUDA graph, and the median replay time over --iters
    replays is divided by --reps, so host enqueue time is excluded; new_kernels_ms is their sum and new_kernels_share its ratio to
    step_graph_ms;
  * profiled_train_kernels_share: torch.profiler's CUDA kernel time of those kernels over the CUDA kernel time of all kernels, over
    --iters eager steps: the share measured inside the step itself.
Prints one JSON document with the GPU name, power limit and maximum SM clock, and writes it to --out when given.
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from hand3d_b200 import autograd as A, runtime, weights as Wt  # noqa: E402
from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork  # noqa: E402
from hand3d_b200.optim import Adam  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"name": name, "power_limit": power, "clocks_max_sm": clock}


def time_ms(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def graph_ms(fn, reps, warmup, iters):
    """GPU time of one fn() call: fn is captured reps times back to back into one CUDA graph (after an eager warm-up on a side
    stream, which also sizes the operator scratch); median replay time / reps."""
    gc.collect()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    ms = time_ms(g.replay, warmup, iters) / reps
    del g
    return ms


# kernel-name fragments of the training kernels (csrc/train.cu) and of the resize forward the step runs on every map
TRAIN_KERNELS = ("resize_bilinear_tf1_kernel", "resize_grad_cols_kernel", "resize_grad_rows_kernel", "scoremap_sq_partial_kernel",
                 "scoremap_loss_finalize_kernel", "scoremap_loss_grad_kernel", "xent_partial_kernel", "xent_finalize_kernel",
                 "xent_grad_kernel", "adam_step_kernel")


def profiled_share(step, iters):
    """(training-kernel CUDA time, all CUDA kernel time) in ms per step, from torch.profiler over iters eager steps."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            step()
        torch.cuda.synchronize()
    train = total = 0.0
    for e in prof.key_averages():
        t = e.self_device_time_total          # microseconds; kernels carry their own time, CPU-side ops none of their own
        total += t
        if any(k in e.key for k in TRAIN_KERNELS):
            train += t
    return train / 1e3 / iters, total / 1e3 / iters


def setup(scope, B, S, seed=0):
    rng = np.random.default_rng(seed)
    img = torch.from_numpy(Wt.synthetic_blob_images(B, S, S, seed=seed)).cuda()
    net = ColorHandPose3DNetwork()
    ctx = runtime.default_context()
    v = ctx.variables(scope)
    opt = Adam(list(v.values()), lr=1e-5)
    if scope == "PoseNet2D":
        target = torch.from_numpy(rng.uniform(size=(B, S, S, 21)).astype(np.float32) * 0.2).cuda()
        vis = torch.from_numpy((rng.uniform(size=(B, 21)) > 0.2).astype(np.float32)).cuda()

        def forward():
            return net.inference_pose2d(img, train=True)

        def loss_of(maps):
            return sum(A.scoremap_loss(A.resize_bilinear(m, S, S), target, vis) for m in maps)
    else:
        hand = img[..., 0] > 0.05
        labels = torch.stack([~hand, hand], 3).to(torch.float32)

        def forward():
            return net.inference_detection(img, train=True)

        def loss_of(maps):
            return A.softmax_xent_loss(maps[0], labels)

    def step():
        opt.zero_grad()
        loss = loss_of(forward())
        loss.backward()
        opt.step()

    return ctx, v, opt, forward, loss_of, step


def bench(scope, B, S, warmup, iters, reps):
    ctx, v, opt, forward, loss_of, step = setup(scope, B, S)
    r = {"net": scope, "B": B, "size": S, "params": int(sum(p.numel() for p in v.values())), "tensors": len(v)}
    r["step_eager_ms"] = time_ms(step, warmup, iters)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            step()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    r["step_graph_ms"] = time_ms(g.replay, warmup, iters)
    del g

    with torch.no_grad():       # no autograd graph may outlive its step: its nodes would be reused on the stream they were made on
        maps = forward()
    grads = [torch.randn_like(m) for m in maps]

    def fwd_bwd():
        torch.autograd.backward(forward(), grads)
    r["net_fwd_bwd_ms"] = graph_ms(fwd_bwd, 2, warmup, iters)

    # the training kernels alone, with the step's shapes
    maps = [m.detach().contiguous() for m in maps]
    up = [ctx.resize_bilinear(m, S, S) for m in maps]
    one = torch.ones((), device="cuda")
    if scope == "PoseNet2D":
        target = torch.rand_like(up[0]) * 0.2
        vis = torch.ones((B, 21), device="cuda")

        def loss_kernels():
            for u in up:
                _, rms = ctx.scoremap_loss(u, target, vis)
                ctx.scoremap_loss_backward(u, target, vis, rms, one)
    else:
        labels = torch.rand_like(up[0])

        def loss_kernels():
            ctx.softmax_xent(up[0], labels)
            ctx.softmax_xent_backward(up[0], labels, one)

    def resize_kernels():
        for m, u in zip(maps, up):
            ctx.resize_bilinear(m, S, S)
            ctx.resize_bilinear_backward(u, m.shape[1], m.shape[2])

    r["resize_fwd_bwd_ms"] = graph_ms(resize_kernels, reps, warmup, iters)
    r["loss_fwd_bwd_ms"] = graph_ms(loss_kernels, reps, warmup, iters)
    r["adam_ms"] = graph_ms(opt.step, reps, warmup, iters)
    r["new_kernels_ms"] = r["resize_fwd_bwd_ms"] + r["loss_fwd_bwd_ms"] + r["adam_ms"]
    r["new_kernels_share"] = r["new_kernels_ms"] / r["step_graph_ms"]
    train_ms, kernels_ms = profiled_share(step, iters)
    r["profiled_train_kernels_ms"], r["profiled_all_kernels_ms"] = train_ms, kernels_ms
    r["profiled_train_kernels_share"] = train_ms / kernels_ms
    return r


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--reps", type=int, default=20, help="back-to-back copies of a kernel group in its timing graph")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    ColorHandPose3DNetwork().init(weights=Wt.synthetic_weights(0))
    runtime.default_context().set_precision("bf16x3")
    doc = {"gpu": gpu_info(), "precision": "bf16x3",
           "results": [bench(s, a.batch, a.size, a.warmup, a.iters, a.reps) for s in ("PoseNet2D", "HandSegNet")]}
    print(json.dumps(doc, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()

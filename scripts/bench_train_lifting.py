"""Times one training step of the lifting stage (training_lifting.py) for each variant on the project's kernels, eagerly and replayed
from a CUDA graph, and splits its GPU time into parts.

Shapes: B = 8 (the reference's batch) and 64 score maps of 256x256x21 (avg-pooled to 32x32 inside the step), hand_side and the
variant's targets.  A step is zero_grad, PosePriorNetwork(variant).inference(train=True), the variant's loss, backward and the Adam
update over the trained scope(s) (both in 'proposed').  Xavier-initialised weights and synthetic inputs: the timings do not depend on
the values.

Reported per variant and batch size (GPU times from CUDA-graph replays as in scripts/bench_train_step.py: each part is captured
--reps times back to back into one graph, median replay time over --iters replays divided by --reps):
  * step_eager_ms, step_graph_ms: the whole step, eagerly and as one replayed CUDA graph;
  * conv_fwd_bwd_ms: the stride-1 / stride-2 convolution pyramids, forward and backward (incoming gradients random);
  * fc_fwd_bwd_ms: the FC stacks on the 1x1 tensor-core convolution, forward and backward;
  * new_kernels_ms: csrc/train_lift.cu's kernels the variant runs (rotate_canonical and its adjoint, the forward kinematics and its
    adjoint, the MSE and its gradient) plus the 8x8 average pool;
  * adam_ms: the Adam step.
Prints one JSON document with the GPU name, power limit and maximum SM clock, and writes it to --out when given.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_train_step import gpu_info, graph_ms, time_ms  # noqa: E402
from hand3d_b200 import arch, autograd as A, runtime, weights as Wt  # noqa: E402
from hand3d_b200.nets.PosePriorNetwork import PosePriorNetwork  # noqa: E402
from hand3d_b200.optim import Adam  # noqa: E402

VARIANTS = ["direct", "bottleneck", "local", "local_w_xyz_loss", "proposed"]


def setup(variant, B, seed=0):
    ctx = runtime.default_context()
    ctx.load_weights(Wt.xavier_weights(seed, bottleneck=variant == "bottleneck"))
    scopes = ["PosePrior", "ViewpointNet"] if variant == "proposed" else ["PosePrior"]
    v = {}
    for s in scopes:
        v.update(ctx.variables(s))
    opt = Adam(list(v.values()), lr=1e-5)
    rng = np.random.default_rng(seed)
    uv = torch.from_numpy(rng.uniform(20, 236, size=(B, 21, 2)).astype(np.float32)).cuda()
    sm = ctx.gaussian_scoremap(uv, (256, 256), 25.0)
    hs = torch.zeros((B, 2), device="cuda")
    hs[torch.arange(B), torch.from_numpy(rng.integers(0, 2, B)).cuda()] = 1
    xyz = torch.from_numpy((rng.normal(size=(B, 21, 3)) * 0.3).astype(np.float32)).cuda()
    can, _, rot = ctx.canonical_trafo(xyz, hs[:, 1] > 0.5)
    local = ctx.bone_rel_trafo(xyz)
    net = PosePriorNetwork(variant)

    def loss_of(coord3d, R):
        if variant in ("direct", "bottleneck"):
            return A.mse_loss(coord3d, xyz)
        if variant == "local":
            return A.mse_loss(coord3d, local)
        if variant == "local_w_xyz_loss":
            return A.mse_loss(A.bone_rel_trafo_inv(coord3d), xyz)
        return A.mse_loss(coord3d, can) + A.mse_loss(R, rot)

    def step():
        opt.zero_grad()
        _, coord3d, R = net.inference(sm, hs, train=True)
        loss_of(coord3d, R).backward()
        opt.step()

    return ctx, v, opt, sm, hs, (xyz, can, rot, local), step


def bench(variant, B, warmup, iters, reps):
    ctx, v, opt, sm, hs, (xyz, can, rot, local), step = setup(variant, B)
    r = {"variant": variant, "B": B, "params": int(sum(p.numel() for p in v.values())), "tensors": len(v)}
    r["step_eager_ms"] = time_ms(step, warmup, iters)
    r["step_graph_ms"] = graph_ms(step, 1, warmup, iters)

    pooled = ctx.avg_pool8(sm)
    scopes = [("PosePrior", arch.POSEPRIOR)] + ([("ViewpointNet", arch.VIEWPOINT)] if variant == "proposed" else [])
    convs, fcs = [], []
    for scope, layers in scopes:
        convs.append((scope, layers[:6]))
        names = ["fc_rel0", "fc_rel1"] + (["fc_bottleneck"] if variant == "bottleneck" else []) + ["fc_xyz"] \
            if scope == "PosePrior" else ["fc_vp0", "fc_vp1", "fc_vp_ux", "fc_vp_uy", "fc_vp_uz"]
        fcs.append((scope, names))

    def conv_fwd():
        outs = []
        for scope, layers in convs:
            x = pooled
            for name, k, stride, _, _, leaky in layers:
                x = A.conv2d(x, v["%s/%s/weights" % (scope, name)], v["%s/%s/biases" % (scope, name)], stride, leaky)
            outs.append(x)
        return outs

    with torch.no_grad():
        conv_dy = [torch.randn_like(o) for o in conv_fwd()]
    r["conv_fwd_bwd_ms"] = graph_ms(lambda: torch.autograd.backward(conv_fwd(), conv_dy), reps, warmup, iters)

    fc_in = {"PosePrior": torch.randn(B, 2050, device="cuda"), "ViewpointNet": torch.randn(B, 4098, device="cuda")}

    def fc_fwd():
        outs = []
        for scope, names in fcs:
            x = fc_in[scope]
            for name in names:
                x = A.fully_connected(x, v["%s/%s/weights" % (scope, name)], v["%s/%s/biases" % (scope, name)],
                                      name in ("fc_rel0", "fc_rel1", "fc_vp0", "fc_vp1"))
                if name == "fc_vp1":
                    break
            outs.append(x)
        if variant == "proposed":        # the three heads as one 128 -> 3 layer, as the train graph runs them
            w = torch.cat([v["ViewpointNet/fc_vp_u%s/weights" % a] for a in "xyz"], 1)
            b = torch.cat([v["ViewpointNet/fc_vp_u%s/biases" % a] for a in "xyz"], 0)
            outs[-1] = A.fully_connected(outs[-1], w, b, False)
        return outs

    with torch.no_grad():
        fc_dy = [torch.randn_like(o) for o in fc_fwd()]
    r["fc_fwd_bwd_ms"] = graph_ms(lambda: torch.autograd.backward(fc_fwd(), fc_dy), reps, warmup, iters)

    one = torch.ones((), device="cuda")
    c = torch.randn(B, 21, 3, device="cuda") * 0.3
    u = torch.randn(B, 3, device="cuda")

    def new_kernels():
        ctx.avg_pool8(sm)
        if variant == "proposed":
            R, _ = ctx.rotate_canonical(c, u, hs)
            ctx.rotate_canonical_backward(c, u, hs, None, ctx.mse_loss_backward(R, rot, one))
            ctx.mse_loss(c, can); ctx.mse_loss(R, rot); ctx.mse_loss_backward(c, can, one)
        elif variant == "local_w_xyz_loss":
            x = ctx.bone_rel_trafo_inv(c)
            ctx.mse_loss(x, xyz)
            ctx.bone_rel_trafo_inv_backward(c, ctx.mse_loss_backward(x, xyz, one))
        else:
            ctx.mse_loss(c, xyz); ctx.mse_loss_backward(c, xyz, one)

    r["new_kernels_ms"] = graph_ms(new_kernels, reps, warmup, iters)
    r["adam_ms"] = graph_ms(opt.step, reps, warmup, iters)
    for k in ("conv_fwd_bwd_ms", "fc_fwd_bwd_ms", "new_kernels_ms", "adam_ms"):
        r[k.replace("_ms", "_share")] = r[k] / r["step_graph_ms"]
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variants", nargs="*", default=VARIANTS)
    ap.add_argument("--batch", type=int, nargs="*", default=[8, 64])
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_lifting.py measures on a CUDA device; none is available")
    runtime.default_context().set_precision("bf16x3")
    doc = {"gpu": gpu_info(), "precision": "bf16x3", "results": []}
    for variant in args.variants:
        for B in args.batch:
            doc["results"].append(bench(variant, B, args.warmup, args.iters, args.reps))
            print(json.dumps(doc["results"][-1]), file=sys.stderr)
    text = json.dumps(doc, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()

"""What the lifting stage's dropout (evaluation=False) costs on the GPU, in one run:

  1. train_step: the graph-replayed lifting training step (scripts/bench_train_lifting.py's step: zero_grad, PosePriorNetwork.inference
     with train=True, the variant's loss, backward, Adam) of all five variants at B = 8 and 64, with evaluation=True and with
     evaluation=False, the two measured alternately --rounds times; the median of each is reported.
  2. lifting_forward: h3d_lifting_forward ('proposed', bf16x3) at B = 32 and 128 with dropout on (the layer-by-layer route with the
     four dropout kernels) against the default fused FC chain, alternately.
  3. kernels: dropout_kernel on fp32 and into bf16 planes, dropout_backward_kernel and the advance kernel at the lifting's shapes.

GPU times are CUDA-graph replays (scripts/bench_train_step.py: graph_ms).  Prints one JSON document with the GPU name, power limit and
maximum SM clock, and writes it to --out when given.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_train_step import gpu_info, graph_ms  # noqa: E402
from hand3d_b200 import autograd as A, runtime, weights as Wt  # noqa: E402
from hand3d_b200.nets.PosePriorNetwork import PosePriorNetwork  # noqa: E402
from hand3d_b200.optim import Adam  # noqa: E402

VARIANTS = ["direct", "bottleneck", "local", "local_w_xyz_loss", "proposed"]


def train_steps(variant, B, seed=0):
    """(step with evaluation=True, step with evaluation=False) over one set of Parameters and one optimiser."""
    ctx = runtime.default_context()
    ctx.load_weights(Wt.xavier_weights(seed, bottleneck=variant == "bottleneck"))
    params = [p for s in (["PosePrior", "ViewpointNet"] if variant == "proposed" else ["PosePrior"]) for p in ctx.variables(s).values()]
    opt = Adam(params, lr=1e-5)
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

    def step(evaluation):
        def run():
            opt.zero_grad()
            _, coord3d, R = net.inference(sm, hs, evaluation=evaluation, train=True)
            loss_of(coord3d, R).backward()
            opt.step()
        return run

    return step(True), step(False)


def alternate(fns, rounds, reps, warmup, iters):
    """Median over `rounds` of graph_ms for each fn, measured fn by fn within a round."""
    ts = [[] for _ in fns]
    for _ in range(rounds):
        for i, fn in enumerate(fns):
            ts[i].append(graph_ms(fn, reps, warmup, iters))
    return [statistics.median(t) for t in ts]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--variants", nargs="*", default=VARIANTS)
    ap.add_argument("--batch", type=int, nargs="*", default=[8, 64])
    ap.add_argument("--lift-batch", type=int, nargs="*", default=[32, 128])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dropout.py measures on a CUDA device; none is available")
    ctx = runtime.default_context()
    ctx.set_precision("bf16x3")
    ctx.set_dropout(2024)
    doc = {"gpu": gpu_info(), "precision": "bf16x3", "train_step": [], "lifting_forward": [], "kernels": []}

    for variant in args.variants:
        for B in args.batch:
            ev, tr = train_steps(variant, B)
            t_ev, t_tr = alternate([ev, tr], args.rounds, 1, args.warmup, args.iters)
            r = {"variant": variant, "B": B, "eval_true_ms": t_ev, "eval_false_ms": t_tr, "dropout_added_us": 1e3 * (t_tr - t_ev)}
            doc["train_step"].append(r)
            print(json.dumps(r), file=sys.stderr)

    ctx.load_weights({k: v for k, v in Wt.synthetic_weights(0).items() if k.startswith(("PosePrior", "ViewpointNet"))})
    for B in args.lift_batch:
        rng = np.random.default_rng(B)
        sm = torch.from_numpy(rng.normal(size=(B, 32, 32, 21)).astype(np.float32)).cuda()
        hs = torch.zeros((B, 2), device="cuda")
        hs[:, 0] = 1
        t_chain, t_drop = alternate([lambda: ctx.lifting(sm, hs, "proposed"), lambda: ctx.lifting(sm, hs, "proposed", dropout=True)],
                                    args.rounds, args.reps, args.warmup, args.iters)
        r = {"B": B, "fused_chain_ms": t_chain, "layers_with_dropout_ms": t_drop}
        doc["lifting_forward"].append(r)
        print(json.dumps(r), file=sys.stderr)

    lib, h = ctx.lib, ctx.h
    for B in args.lift_batch:
        for cols in (512, 256, 128):
            x = torch.randn(B, cols, device="cuda")
            keep = torch.empty((B, cols), dtype=torch.uint8, device="cuda")
            hi = torch.empty((B, cols), dtype=torch.int16, device="cuda")
            lo = torch.empty_like(hi)
            y = torch.empty_like(x)
            s = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)   # noqa: E731
            p = lambda t: C.c_void_p(t.data_ptr())                              # noqa: E731
            ctx._dropout_mode(True)
            fns = {
                "forward_f32": lambda: lib.h3d_dropout_forward(h, p(x), B, cols, 0.8, 0, p(y), p(keep), s()),
                "forward_planes": lambda: lib.h3d_dropout_forward_planes(h, p(x), B, cols, 0.8, 0, None, None, 0, cols, p(hi), p(lo), s()),
                "backward": lambda: lib.h3d_dropout_backward(h, p(x), p(keep), B, cols, 0.8, p(y), s()),
                "advance": lambda: lib.h3d_dropout_advance(h, s()),
            }
            r = {"B": B, "cols": cols}
            for name, fn in fns.items():
                r[name + "_us"] = 1e3 * graph_ms(fn, 20, args.warmup, args.iters)
            doc["kernels"].append(r)
            print(json.dumps(r), file=sys.stderr)
    ctx.set_dropout(None)
    text = json.dumps(doc, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()

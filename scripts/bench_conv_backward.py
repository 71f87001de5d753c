"""Times the tensor-core convolution's forward, data gradient and weight gradient per layer, against torch/cuDNN in fp32 (TF32 off).

Layers: every convolution of PoseNet2D at the reference's training batch (B = 8 crops of 256x256, training_posenet.py:38) and of
HandSegNet at 320x320 (B = 8), with the spatial sizes the max-pools give.  Per layer and operation the median of --iters CUDA-event
timings after --warmup untimed runs, the algorithmic TFLOP/s (2 B Ho Wo k^2 Cin Cout with the real, unpadded channel counts, as
hand3d_b200/arch.py counts them) and the (dx + dW) / forward ratio.  The data gradient of a first layer (Cin = 3) is not timed: a
training step never needs it.  The forward is h3d_conv2d_tc_dev (device weights packed every call, as a training step runs it);
each gradient time includes the dy' preparation pass.  Last, forward + backward of the PoseNet2D trunk (conv1_1 .. conv5_2 with
its three max-pools) through hand3d_b200.autograd.

Prints one JSON document (with the GPU name, power limit and maximum SM clock read in the same run) and writes it to --out when
given.  Needs an sm_90a GPU; there is no fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from hand3d_b200 import arch, autograd, runtime  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"name": name, "power_limit": power, "clocks_max_sm": clock}


def layers(B=8):
    """(net, name, B, H, W, k, Cin, Cout, leaky) of every convolution, at the resolution it runs."""
    out = []
    for net, table, size, pools in (("PoseNet2D", arch.POSENET2D, 256, arch.POSENET2D_POOL_AFTER),
                                    ("HandSegNet", arch.HANDSEGNET, 320, arch.HANDSEGNET_POOL_AFTER)):
        h = size
        for name, k, s, cin, cout, leaky in table:
            out.append((net, name, B, h, h, k, cin, cout, leaky))
            if name in pools:
                h //= 2
    return out


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


def bench_layer(ctx, layer, precision, warmup, iters):
    net, name, B, H, W, k, cin, cout, leaky = layer
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn((B, H, W, cin), device="cuda", generator=g)
    w = torch.randn((k, k, cin, cout), device="cuda", generator=g) / (k * k * cin) ** 0.5
    b = torch.randn((cout,), device="cuda", generator=g) * 0.1
    dy = torch.randn((B, H, W, cout), device="cuda", generator=g)
    y = ctx.conv2d_tc_dev(x, w, b, leaky=leaky, precision=precision)
    first = cin == 3
    flops = 2.0 * B * H * W * k * k * cin * cout
    r = {"net": net, "layer": name, "B": B, "H": H, "W": W, "k": k, "cin": cin, "cout": cout, "gflop": flops / 1e9}
    r["fwd_ms"] = time_ms(lambda: ctx.conv2d_tc_dev(x, w, b, leaky=leaky, precision=precision), warmup, iters)
    r["dx_ms"] = None if first else time_ms(lambda: ctx.conv2d_tc_backward(x, y, dy, w, leaky=leaky, precision=precision, need_dw=False,
                                                                          need_db=False), warmup, iters)
    r["dw_ms"] = time_ms(lambda: ctx.conv2d_tc_backward(x, y, dy, w, leaky=leaky, precision=precision, need_dx=False, need_db=True),
                         warmup, iters)
    # torch / cuDNN yardstick on the same shapes, fp32 without TF32 (NCHW views of the channels-last tensors)
    xc, wc, dyc = x.permute(0, 3, 1, 2), w.permute(3, 2, 0, 1).contiguous(memory_format=torch.channels_last), dy.permute(0, 3, 1, 2)
    p = k // 2
    r["cudnn_fwd_ms"] = time_ms(lambda: F.conv2d(xc, wc, b, padding=p), warmup, iters)
    r["cudnn_dx_ms"] = None if first else time_ms(lambda: torch.nn.grad.conv2d_input(xc.shape, wc, dyc, padding=p), warmup, iters)
    r["cudnn_dw_ms"] = time_ms(lambda: torch.nn.grad.conv2d_weight(xc, wc.shape, dyc, padding=p), warmup, iters)
    for key in ("fwd", "dx", "dw", "cudnn_fwd", "cudnn_dx", "cudnn_dw"):
        ms = r[key + "_ms"]
        r[key + "_tflops"] = None if ms is None else flops / (ms * 1e-3) / 1e12
    r["bwd_over_fwd"] = ((r["dx_ms"] or 0.0) + r["dw_ms"]) / r["fwd_ms"]
    return r


def bench_trunk(precision, warmup, iters, B=8, size=256):
    """forward + backward of PoseNet2D conv1_1 .. conv5_2 through autograd.py (loss = <output, g>)."""
    g = torch.Generator(device="cuda").manual_seed(1)
    params, plan = [], []
    for name, k, s, cin, cout, leaky in arch.POSENET2D:
        params += [torch.nn.Parameter(torch.randn((k, k, cin, cout), device="cuda", generator=g) / (k * k * cin) ** 0.5),
                   torch.nn.Parameter(torch.randn((cout,), device="cuda", generator=g) * 0.1)]
        plan.append((leaky, name in arch.POSENET2D_POOL_AFTER))
        if name == "conv5_2":
            break
    x = torch.randn((B, size, size, 3), device="cuda", generator=g)
    go = torch.randn((B, size // 8, size // 8, 21), device="cuda", generator=g)

    def step():
        h = x
        for i, (leaky, pool) in enumerate(plan):
            h = autograd.conv2d(h, params[2 * i], params[2 * i + 1], leaky=leaky, precision=precision)
            if pool:
                h = autograd.max_pool(h)
        (h * go).sum().backward()

    ms = time_ms(step, warmup, iters)
    return {"layers": "PoseNet2D conv1_1..conv5_2", "B": B, "size": size, "fwd_bwd_ms": ms}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--precision", default="bf16x3", choices=["bf16x3", "bf16"])
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON document here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_conv_backward.py needs an sm_90a GPU")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    ctx = runtime.default_context()
    res = {"gpu": gpu_info(), "precision": args.precision, "layers": [], "trunk": None}
    for layer in layers():
        r = bench_layer(ctx, layer, args.precision, args.warmup, args.iters)
        res["layers"].append(r)
        print("%-10s %-8s %3dx%-3d k%d %3d->%-3d fwd %7.3f ms  dx %7s  dW %7.3f ms  (bwd/fwd %.2f)   cuDNN fp32: fwd %7.3f dx %7s dW %7.3f"
              % (r["net"], r["layer"], r["H"], r["W"], r["k"], r["cin"], r["cout"], r["fwd_ms"],
                 "-" if r["dx_ms"] is None else "%.3f" % r["dx_ms"], r["dw_ms"], r["bwd_over_fwd"], r["cudnn_fwd_ms"],
                 "-" if r["cudnn_dx_ms"] is None else "%.3f" % r["cudnn_dx_ms"], r["cudnn_dw_ms"]), file=sys.stderr)
    res["trunk"] = bench_trunk(args.precision, args.warmup, args.iters)
    for net in ("PoseNet2D", "HandSegNet"):
        rows = [r for r in res["layers"] if r["net"] == net]
        tot = {k: sum((r[k] or 0.0) for r in rows) for k in ("fwd_ms", "dx_ms", "dw_ms", "cudnn_fwd_ms", "cudnn_dx_ms", "cudnn_dw_ms")}
        tot["bwd_over_fwd"] = (tot["dx_ms"] + tot["dw_ms"]) / tot["fwd_ms"]
        res[net + "_total"] = tot
    doc = json.dumps(res, indent=1)
    print(doc)
    if args.out:
        with open(args.out, "w") as f:
            f.write(doc)


if __name__ == "__main__":
    main()

"""torch.autograd functions over the tensor-core convolution and the max-pool, so that a plain torch.optim loop can train through
the project's own kernels (the gradients TF's AdamOptimizer.minimize evaluates in training_posenet.py:67 / training_handsegnet.py).

Tensors are NHWC float32 on a CUDA device; `w` is an HWIO Parameter shaped like the reference variable ([k,k,Cin,Cout], as in
weights.synthetic_weights() or a loaded pickle) and `b` a [Cout] Parameter.  Forward and backward run on the default Context of the
input's device; there is no CPU path.

    y = conv2d(x, w, b, stride=1, leaky=True)    # NetworkOps.conv_relu (leaky=False: NetworkOps.conv)
    p = max_pool(y)                              # NetworkOps.max_pool
"""
from __future__ import annotations

import torch

from . import runtime


def _ctx(t):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError("hand3d_b200.autograd works on CUDA tensors only (there is no CPU path)")
    return runtime.default_context(t.device)


class _Conv2d(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, stride, leaky, precision):
        h = _ctx(x)
        y = h.conv2d_tc_dev(x, w.detach(), b.detach(), stride=stride, leaky=leaky, precision=precision)
        ctx.save_for_backward(x, w, y if leaky else None)
        ctx.conf = (stride, leaky, precision)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, y = ctx.saved_tensors
        stride, leaky, precision = ctx.conf
        need_dx, need_dw, need_db = ctx.needs_input_grad[:3]
        if not (need_dx or need_dw or need_db):
            return None, None, None, None, None, None
        dx, dw, db = _ctx(dy).conv2d_tc_backward(x, y, dy, w.detach(), stride=stride, leaky=leaky, precision=precision,
                                                 need_dx=need_dx, need_dw=need_dw, need_db=need_db)
        return dx, dw, db, None, None, None


class _MaxPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        y = _ctx(x).max_pool(x)
        ctx.save_for_backward(x)
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        return _ctx(dy).max_pool_backward(x, dy)


def conv2d(x, w, b, stride=1, leaky=True, precision="bf16x3"):
    """act(conv_SAME(x, w, stride) + b) on the wgmma kernels.  stride 1, or 2 with even H, W and k >= 3; k in {1, 3, 5, 7}.
    The backward supports precision "bf16x3" (fp32 parity) and "bf16"."""
    return _Conv2d.apply(x, w, b, int(stride), bool(leaky), precision)


def max_pool(x):
    """2x2 / 2 VALID max-pool; the gradient goes to the first maximum of each window (row-major), as TF's MaxPoolGrad."""
    return _MaxPool.apply(x)

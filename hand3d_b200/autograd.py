"""torch.autograd functions over the tensor-core convolution and the max-pool, so that a plain torch.optim loop can train through
the project's own kernels (the gradients TF's AdamOptimizer.minimize evaluates in training_posenet.py:67 / training_handsegnet.py).

Tensors are NHWC float32 on a CUDA device; `w` is an HWIO Parameter shaped like the reference variable ([k,k,Cin,Cout], as in
weights.synthetic_weights() or a loaded pickle) and `b` a [Cout] Parameter.  Forward and backward run on the default Context of the
input's device; there is no CPU path.

    y = conv2d(x, w, b, stride=1, leaky=True)    # NetworkOps.conv_relu (leaky=False: NetworkOps.conv)
    p = max_pool(y)                              # NetworkOps.max_pool
    u = resize_bilinear(s, 256, 256)             # tf.image.resize_images
    L = scoremap_loss(u, target, vis)            # training_posenet.py:61, one map
    L = softmax_xent_loss(logits, labels)        # training_handsegnet.py:60

The backward of every function reads the incoming gradient on the device: no .item(), no host synchronisation, so a whole training
step can be captured into a CUDA graph.
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


class _Resize(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, out_h, out_w):
        ctx.in_hw = (x.shape[1], x.shape[2])
        return _ctx(x).resize_bilinear(x, out_h, out_w)

    @staticmethod
    def backward(ctx, dy):
        return _ctx(dy).resize_bilinear_backward(dy, *ctx.in_hw), None, None


class _ScoremapLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, target, vis):
        loss, rms = _ctx(pred).scoremap_loss(pred, target, vis)
        ctx.save_for_backward(pred, target, vis, rms)
        return loss

    @staticmethod
    def backward(ctx, g):
        pred, target, vis, rms = ctx.saved_tensors
        return _ctx(g).scoremap_loss_backward(pred, target, vis, rms, g), None, None


class _SoftmaxXent(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, labels):
        ctx.save_for_backward(logits, labels)
        return _ctx(logits).softmax_xent(logits, labels)

    @staticmethod
    def backward(ctx, g):
        logits, labels = ctx.saved_tensors
        return _ctx(g).softmax_xent_backward(logits, labels, g), None


def resize_bilinear(x, out_h, out_w):
    """tf.image.resize_images (bilinear, align_corners=False, TF1 legacy) of x [B,H,W,C]; the backward is the forward's exact adjoint
    (ResizeBilinearGrad)."""
    return _Resize.apply(x, int(out_h), int(out_w))


def scoremap_loss(pred, target, vis):
    """training_posenet.py:61 for one map: sum vis sqrt(mean_hw (pred - target)^2) / (sum vis + 0.001); pred, target [B,H,W,21],
    vis [B,21] (any dtype, cast to fp32).  Only pred receives a gradient; it is 0 where a (b, k) map matches its target exactly."""
    return _ScoremapLoss.apply(pred, target.detach(), vis.detach().to(torch.float32))


def softmax_xent_loss(logits, labels):
    """training_handsegnet.py:60: reduce_mean(softmax_cross_entropy_with_logits(logits, labels)) over every [..., 2] row; labels fp32
    (not necessarily one-hot).  Only logits receive a gradient."""
    return _SoftmaxXent.apply(logits, labels.detach().to(torch.float32))


def conv2d(x, w, b, stride=1, leaky=True, precision="bf16x3"):
    """act(conv_SAME(x, w, stride) + b) on the wgmma kernels.  stride 1, or 2 with even H, W and k >= 3; k in {1, 3, 5, 7}.
    The backward supports precision "bf16x3" (fp32 parity) and "bf16"."""
    return _Conv2d.apply(x, w, b, int(stride), bool(leaky), precision)


def max_pool(x):
    """2x2 / 2 VALID max-pool; the gradient goes to the first maximum of each window (row-major), as TF's MaxPoolGrad."""
    return _MaxPool.apply(x)

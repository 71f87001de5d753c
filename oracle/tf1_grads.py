"""fp64 restatement of the TF 1.x gradient kernels AdamOptimizer.minimize evaluates through NetworkOps.conv / conv_relu / max_pool
(training_posenet.py:67, training_handsegnet.py): Conv2DBackpropInput, Conv2DBackpropFilter, BiasAddGrad, the Maximum gradient of
tf.maximum(x, 0.01 x) and the CPU MaxPoolGrad.

Test-only, like tf1_ops: numpy / torch-CPU arrays in NHWC with HWIO weights, computed in float64.  'SAME' padding is TF's (tf1_ops.same_pad:
for stride 2 on an even size, 0 before and 1 after, or 1 / 2 for k = 5 ...), written out as explicit index arithmetic rather than a
library transposed convolution.
"""
from __future__ import annotations

import numpy as np
import torch

from .tf1_ops import NEG_SLOPE, same_pad


def _t64(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64))


def conv2d_backprop_input(dy, w, x_shape, stride=1):
    """tf.nn.conv2d_backprop_input: dx[b, oy s + kh - pt, ox s + kw - pl, ci] += dy[b, oy, ox, co] w[kh, kw, ci, co]."""
    B, H, W, Cin = x_shape
    k = w.shape[0]
    pt, _ = same_pad(H, k, stride)
    pl, _ = same_pad(W, k, stride)
    dy, w = _t64(dy), _t64(w)
    Ho, Wo = dy.shape[1], dy.shape[2]
    Hp, Wp = (Ho - 1) * stride + k, (Wo - 1) * stride + k
    dxp = torch.zeros((B, Hp, Wp, Cin), dtype=torch.float64)
    for kh in range(k):
        for kw in range(k):
            dxp[:, kh:kh + (Ho - 1) * stride + 1:stride, kw:kw + (Wo - 1) * stride + 1:stride, :] += dy @ w[kh, kw].T
    return dxp[:, pt:pt + H, pl:pl + W, :].numpy()


def conv2d_backprop_filter(x, dy, k, stride=1):
    """tf.nn.conv2d_backprop_filter: dw[kh, kw, ci, co] = sum_{b, oy, ox} x[b, oy s + kh - pt, ox s + kw - pl, ci] dy[b, oy, ox, co]."""
    B, H, W, Cin = x.shape
    pt, pb = same_pad(H, k, stride)
    pl, pr = same_pad(W, k, stride)
    dy = _t64(dy)
    Ho, Wo, Cout = dy.shape[1], dy.shape[2], dy.shape[3]
    xp = torch.zeros((B, H + pt + pb + k, W + pl + pr + k, Cin), dtype=torch.float64)
    xp[:, pt:pt + H, pl:pl + W, :] = _t64(x)
    dyf = dy.reshape(-1, Cout)
    dw = torch.zeros((k, k, Cin, Cout), dtype=torch.float64)
    for kh in range(k):
        for kw in range(k):
            xs = xp[:, kh:kh + (Ho - 1) * stride + 1:stride, kw:kw + (Wo - 1) * stride + 1:stride, :].reshape(-1, Cin)
            dw[kh, kw] = xs.T @ dyf
    return dw.numpy()


def bias_add_grad(dy):
    """tf.nn.bias_add gradient: the sum of dy over every axis but the channel."""
    return _t64(dy).sum(dim=(0, 1, 2)).numpy()


def leaky_relu_grad(pre, dy):
    """Gradient of tf.maximum(pre, 0.01 pre) (utils/general.py:31-33): TF's Maximum gradient routes dy to the first argument where
    pre >= 0.01 pre, to the second (then through the multiply by 0.01) elsewhere."""
    pre, dy = np.asarray(pre, np.float64), np.asarray(dy, np.float64)
    first = pre >= NEG_SLOPE * pre
    return np.where(first, dy, 0.0) + NEG_SLOPE * np.where(first, 0.0, dy)


def conv_grads(x, w, b, dy, stride=1, leaky=True, pre=None):
    """(dx, dw, db) of act(conv2d_same(x, w, stride) + b) for the upstream gradient dy, all fp64.  pre: the activation's input (or its
    output, which has the same sign), computed here in fp64 when not given."""
    k = w.shape[0]
    if leaky:
        if pre is None:
            from .tf1_ops import conv2d_same
            pre = conv2d_same(np.asarray(x, np.float64), np.asarray(w, np.float64), np.asarray(b, np.float64), stride, np.float64)
        dy = leaky_relu_grad(pre, dy)
    return conv2d_backprop_input(dy, w, x.shape, stride), conv2d_backprop_filter(x, dy, k, stride), bias_add_grad(dy)


def max_pool_grad(x, dy):
    """TF CPU MaxPoolGrad for the 2x2 / 2 VALID pool: each window's dy goes to its first maximum in row-major window order; rows and
    columns the VALID pool drops get zero."""
    x = np.asarray(x, np.float64)
    B, H, W, C = x.shape
    Ho, Wo = H // 2, W // 2
    win = x[:, :2 * Ho, :2 * Wo, :].reshape(B, Ho, 2, Wo, 2, C).transpose(0, 1, 3, 2, 4, 5).reshape(B, Ho, Wo, 4, C)
    arg = np.argmax(win, axis=3)   # numpy returns the first occurrence of the maximum
    g = np.zeros((B, Ho, Wo, 4, C))
    np.put_along_axis(g, arg[:, :, :, None, :], np.asarray(dy, np.float64)[:, :, :, None, :], axis=3)
    dx = np.zeros((B, H, W, C))
    dx[:, :2 * Ho, :2 * Wo, :] = g.reshape(B, Ho, Wo, 2, 2, C).transpose(0, 1, 3, 2, 4, 5).reshape(B, 2 * Ho, 2 * Wo, C)
    return dx

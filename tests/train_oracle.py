"""fp64 restatement of what TF 1.3 evaluates in training_posenet.py / training_handsegnet.py beyond the convolution gradients
(oracle/tf1_grads.py): ResizeBilinearGrad (legacy, align_corners=False), the PoseNet score-map loss and the HandSegNet softmax
cross-entropy with their gradients, and ApplyAdam, the last also as a float32 restatement in TF's operation order.

Test-only: numpy / torch-CPU, NHWC.  The resize's source indices and weights come from the legacy formula evaluated in `index_dtype`
(float32 as TF and the device compute them; float64 to match oracle/tf1_ops.resize_bilinear_tf1 on fp64 input exactly).
"""
from __future__ import annotations

import numpy as np
import torch


def resize_axis_matrix(n_in, n_out, index_dtype=np.float32):
    """A [n_out, n_in] with out = A @ in along one axis: row o has (1 - l) at i0 and l at i1 (both on i0 == i1 at a clamped edge)."""
    if n_in == n_out:
        return np.eye(n_in)
    ft = np.dtype(index_dtype).type
    scale = ft(n_in) / ft(n_out)
    src = np.arange(n_out, dtype=index_dtype) * scale
    i0 = np.floor(src).astype(np.int64)
    i1 = np.minimum(i0 + 1, n_in - 1)
    lam = (src - i0.astype(index_dtype)).astype(np.float64)
    A = np.zeros((n_out, n_in))
    np.add.at(A, (np.arange(n_out), i0), 1.0 - lam)
    np.add.at(A, (np.arange(n_out), i1), lam)
    return A


def resize_bilinear(x, out_h, out_w, index_dtype=np.float32):
    """The legacy bilinear resize as the linear map it is, in fp64: y[b] = Ay x[b] Axᵀ per channel."""
    x = np.asarray(x, np.float64)
    if x.shape[1:3] == (out_h, out_w):
        return x.copy()
    Ay, Ax = resize_axis_matrix(x.shape[1], out_h, index_dtype), resize_axis_matrix(x.shape[2], out_w, index_dtype)
    return np.einsum("oh,bhwc,pw->bopc", Ay, x, Ax)


def resize_bilinear_grad(dy, H, W, index_dtype=np.float32):
    """TF ResizeBilinearGrad: dx = Ayᵀ dy Ax, the adjoint of resize_bilinear (a copy when the size does not change)."""
    dy = np.asarray(dy, np.float64)
    if dy.shape[1:3] == (H, W):
        return dy.copy()
    Ay, Ax = resize_axis_matrix(H, dy.shape[1], index_dtype), resize_axis_matrix(W, dy.shape[2], index_dtype)
    return np.einsum("oh,bopc,pw->bhwc", Ay, dy, Ax)


def resize_bilinear_torch(x, out_h, out_w, index_dtype=np.float32):
    """The same forward as a differentiable torch expression of gathers and lerps (for torch.autograd)."""
    B, H, W, C = x.shape
    if (H, W) == (out_h, out_w):
        return x

    def axis(n_in, n_out):
        ft = np.dtype(index_dtype).type
        src = np.arange(n_out, dtype=index_dtype) * (ft(n_in) / ft(n_out))
        i0 = np.floor(src).astype(np.int64)
        return torch.from_numpy(i0), torch.from_numpy(np.minimum(i0 + 1, n_in - 1)), torch.from_numpy((src - i0).astype(np.float64))

    y0, y1, ly = axis(H, out_h)
    x0, x1, lx = axis(W, out_w)
    r0, r1 = x[:, y0], x[:, y1]
    lx = lx.to(x.dtype).reshape(1, 1, out_w, 1)
    top = r0[:, :, x0] + (r0[:, :, x1] - r0[:, :, x0]) * lx
    bot = r1[:, :, x0] + (r1[:, :, x1] - r1[:, :, x0]) * lx
    return top + (bot - top) * ly.to(x.dtype).reshape(1, out_h, 1, 1)


# ---- PoseNet score-map loss (training_posenet.py:58-61), one map ---------------------------------------------------------------
def scoremap_loss(P, T, vis):
    P, T, vis = (np.asarray(a, np.float64) for a in (P, T, vis))
    rms = np.sqrt(np.mean((P - T) ** 2, axis=(1, 2)))            # [B,21]
    return float(np.sum(vis * rms) / (np.sum(vis) + 0.001)), rms


def scoremap_loss_grad(P, T, vis, g=1.0):
    """dL/dP = g vis / S (P - T) / (H W rms); 0 where rms == 0 (the library's choice where TF gives NaN)."""
    P, T, vis = (np.asarray(a, np.float64) for a in (P, T, vis))
    _, rms = scoremap_loss(P, T, vis)
    H, W = P.shape[1:3]
    S = np.sum(vis) + 0.001
    with np.errstate(divide="ignore", invalid="ignore"):
        coef = np.where(rms > 0, g * vis / S / (H * W * rms), 0.0)
    return coef[:, None, None, :] * (P - T)


def scoremap_loss_torch(P, T, vis):
    return torch.sum(vis * torch.sqrt(torch.mean((P - T) ** 2, dim=(1, 2)))) / (torch.sum(vis) + 0.001)


# ---- HandSegNet loss (training_handsegnet.py:56-60) -------------------------------------------------------------------------
def softmax_xent(logits, labels):
    """mean over rows of sum labels (lse - (x - m)), rows of the last axis (2 classes)."""
    x, l = np.asarray(logits, np.float64).reshape(-1, 2), np.asarray(labels, np.float64).reshape(-1, 2)
    sh = x - x.max(1, keepdims=True)
    lse = np.log(np.exp(sh).sum(1, keepdims=True))
    return float(np.mean(np.sum(l * (lse - sh), 1)))


def softmax_xent_grad(logits, labels, g=1.0):
    """TF's backprop g / N (softmax - labels): the derivative of softmax_xent only where every label row sums to 1."""
    x, l = np.asarray(logits, np.float64), np.asarray(labels, np.float64)
    e = np.exp(x - x.max(-1, keepdims=True))
    n = x.size // 2
    return g / n * (e / e.sum(-1, keepdims=True) - l)


def softmax_xent_torch(logits, labels):
    return torch.mean(torch.sum(-labels * torch.log_softmax(logits, -1), -1))


# ---- ApplyAdam (TF 1.3 training_ops.cc) -------------------------------------------------------------------------------------
def adam_tf_f32(p, g, m, v, lr, beta1_power, beta2_power, beta1=0.9, beta2=0.999, epsilon=1e-8):
    """One step in float32, in TF's operation order (every intermediate rounded to float32, no FMA).  Returns new (p, m, v)."""
    f = np.float32
    p, g, m, v = (np.asarray(a, f) for a in (p, g, m, v))
    lr, b1p, b2p, b1, b2, eps = (f(a) for a in (lr, beta1_power, beta2_power, beta1, beta2, epsilon))
    alpha = f(f(lr * f(np.sqrt(f(f(1) - b2p)))) / f(f(1) - b1p))
    m = (m + ((g - m) * f(f(1) - b1)).astype(f)).astype(f)
    v = (v + ((g * g).astype(f) - v).astype(f) * f(f(1) - b2)).astype(f)
    p = (p - ((m * alpha).astype(f) / (np.sqrt(v).astype(f) + eps).astype(f)).astype(f)).astype(f)
    return p, m, v


def adam_tf_f64(p, g, m, v, lr, beta1_power, beta2_power, beta1=0.9, beta2=0.999, epsilon=1e-8):
    p, g, m, v = (np.asarray(a, np.float64) for a in (p, g, m, v))
    alpha = lr * np.sqrt(1 - beta2_power) / (1 - beta1_power)
    m = m + (g - m) * (1 - beta1)
    v = v + (g * g - v) * (1 - beta2)
    return p - m * alpha / (np.sqrt(v) + epsilon), m, v


def beta_powers_after(t, beta1=0.9, beta2=0.999):
    """(beta1^(t+1), beta2^(t+1)) as AdamOptimizer._finish accumulates them in float32 from beta1, beta2 over t steps."""
    f = np.float32
    b1p, b2p = f(beta1), f(beta2)
    for _ in range(t):
        b1p, b2p = f(b1p * f(beta1)), f(b2p * f(beta2))
    return b1p, b2p

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
    y = fully_connected(x, w, b, leaky=True)     # ops.fully_connected_relu, on the 1x1 tensor-core convolution
    R, out = rotate_canonical(can, uxyz, hs)     # PosePriorNetwork 'proposed': Rodrigues, flip, rotate
    xyz = bone_rel_trafo_inv(rel)                # the 'local*' variants' forward kinematics
    L = mse_loss(pred, target)                   # training_lifting.py:63-76
    y = dropout(x, 0.8, layer)                   # ops.dropout with evaluation=False, on a seeded context (Context.set_dropout)

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


class _RotateCanonical(torch.autograd.Function):
    @staticmethod
    def forward(ctx, can, uxyz, hand_side):
        ctx.set_materialize_grads(False)        # an unused output passes None, and the kernel skips its term
        ctx.save_for_backward(can, uxyz, hand_side)
        return _ctx(can).rotate_canonical(can, uxyz, hand_side)

    @staticmethod
    def backward(ctx, d_rot, d_out):
        can, uxyz, hand_side = ctx.saved_tensors
        if d_rot is None and d_out is None:
            return None, None, None
        d_can, d_u = _ctx(can).rotate_canonical_backward(can, uxyz, hand_side, d_out, d_rot)
        return d_can, d_u, None


class _BoneRelTrafoInv(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rel):
        ctx.save_for_backward(rel)
        return _ctx(rel).bone_rel_trafo_inv(rel)

    @staticmethod
    def backward(ctx, d_xyz):
        (rel,) = ctx.saved_tensors
        return _ctx(d_xyz).bone_rel_trafo_inv_backward(rel, d_xyz).reshape(rel.shape)


class _MseLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, target):
        ctx.save_for_backward(pred, target)
        return _ctx(pred).mse_loss(pred, target)

    @staticmethod
    def backward(ctx, g):
        pred, target = ctx.saved_tensors
        return _ctx(g).mse_loss_backward(pred, target, g), None


class _Dropout(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, keep_prob, layer):
        y, keep = _ctx(x).dropout_forward(x, keep_prob, layer)
        ctx.save_for_backward(keep)
        ctx.keep_prob = keep_prob
        return y

    @staticmethod
    def backward(ctx, dy):
        (keep,) = ctx.saved_tensors
        return _ctx(dy).dropout_backward(dy.contiguous(), keep, ctx.keep_prob), None, None


def dropout(x, keep_prob, layer):
    """TF 1.3 dropout (utils/general.py:139-148) of x [rows, ...] at the context's current draw, with `layer` as the generator's layer id
    (H3D_DROPOUT_LAYER_*): y = (x / keep_prob) * k.  The keep bits are saved for the backward, dx = (dy * k) / keep_prob.  Does not
    advance the draw: Context.dropout_advance() does, once per network forward."""
    return _Dropout.apply(x.contiguous(), float(keep_prob), int(layer))


def fully_connected(x, w, b, leaky=True, precision="bf16x3"):
    """ops.fully_connected(_relu) (utils/general.py:113-137): act(x w + b) for x [B,in], w [in,out], b [out], run as the 1x1
    tensor-core convolution of x viewed as [B,1,1,in] (the layout the inference FC layers use); leaky=False is the plain layer."""
    B, n_in = x.shape
    y = conv2d(x.contiguous().view(B, 1, 1, n_in), w.view(1, 1, *w.shape), b, 1, leaky, precision)
    return y.view(B, w.shape[1])


def rotate_canonical(can, uxyz, hand_side):
    """The end of the 'proposed' lifting (nets/PosePriorNetwork.py:82-91): R = Rodrigues(uxyz) [B,3,3], out = flip(can) R [B,21,3],
    z mirrored where argmax(hand_side) == 1.  Returns (R, out); can and uxyz receive gradients from either output."""
    return _RotateCanonical.apply(can.contiguous(), uxyz.contiguous(), hand_side.detach().to(torch.float32).contiguous())


def bone_rel_trafo_inv(coords_rel):
    """utils/relative_trafo.py:243-295 with its adjoint: coords_rel [B,21,3] (length, angle_x, angle_y) -> xyz [B,21,3]."""
    return _BoneRelTrafoInv.apply(coords_rel.contiguous())


def mse_loss(pred, target):
    """tf.reduce_mean(tf.square(pred - target)) (training_lifting.py:63-76) over any shape; only pred receives a gradient."""
    return _MseLoss.apply(pred.contiguous(), target.detach().to(torch.float32).contiguous())


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

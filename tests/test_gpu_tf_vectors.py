"""TensorFlow's own op-test vectors (see tests/test_tf_published_vectors.py for sources) run through the CUDA kernels via the
C ABI: the device code is held to tables the builder of neither the kernels nor the oracle wrote."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_tf_published_vectors import TF_CONV_SAME, TF_CROP, TF_RESIZE, _seq  # noqa: E402

pytestmark = pytest.mark.gpu
f32 = np.float32


@pytest.fixture(scope="module")
def ctx():
    from hand3d_b200 import runtime
    return runtime.default_context()


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=f32)).cuda()


@pytest.mark.parametrize("case", TF_CONV_SAME, ids=[c[0] for c in TF_CONV_SAME])
def test_tf_conv2d_same_vectors_fp32_kernel(ctx, case):
    """conv_ops_test.py tables through conv_direct_kernel (h3d_conv2d_f32): SAME padding incl. the stride-2 / stride-3 cases,
    HWIO weights, cross-correlation.  Integer-valued inputs: the fp32 result is exact."""
    _, xs, ws, stride, expected = case
    y = ctx.conv2d(_cuda(_seq(xs)), _cuda(_seq(ws)), _cuda(np.zeros(ws[3], f32)), stride=stride).cpu().numpy()
    np.testing.assert_array_equal(y.reshape(-1), np.array(expected, f32))


def test_tf_conv2d_1x1_vector_tensor_core_kernel(ctx):
    """testConv2D1x1Filter through the wgmma implicit-GEMM kernel (channels zero-padded 3 -> 64 on both sides): small
    integers are exact in bf16 hi/lo split arithmetic."""
    _, xs, ws, _, expected = TF_CONV_SAME[0]
    y = ctx.conv2d_tc(_cuda(_seq(xs)), _seq(ws), np.zeros(ws[3], f32), leaky=False, precision="bf16x3").cpu().numpy()
    np.testing.assert_array_equal(y.reshape(-1), np.array(expected, f32))


def test_tf_conv2d_3x3_same_integer_table_tensor_core_kernel(ctx):
    """3x3 SAME on the tensor-core kernel against the exact integer result (same construction as TF's tables: 1, 2, 3, ...)."""
    from oracle import tf1_ops as T
    x = (_seq((1, 6, 5, 4)) % 13).astype(f32); w = (_seq((3, 3, 4, 8)) % 7 - 3).astype(f32)
    ref = T.conv2d_same(x, w, np.zeros(8, f32), 1, np.float64)
    for stride in (1, 2):
        xi = x if stride == 1 else np.concatenate([x, x[:, :, :1]], 2)     # stride 2 needs even sizes: 6 x 6
        r = T.conv2d_same(xi, w, np.zeros(8, f32), stride, np.float64)
        y = ctx.conv2d_tc(_cuda(xi), w, np.zeros(8, f32), leaky=False, precision="bf16x3", stride=stride).cpu().numpy()
        np.testing.assert_array_equal(y, r.astype(f32))
    assert ref.shape == (1, 6, 5, 8)


@pytest.mark.parametrize("case", TF_RESIZE, ids=[c[0] for c in TF_RESIZE])
def test_tf_resize_bilinear_vectors(ctx, case):
    _, ishape, oshape, data, expected = case
    x = np.array(data, f32).reshape(1, ishape[0], ishape[1], 1)
    y = ctx.resize_bilinear(_cuda(x), oshape[0], oshape[1]).cpu().numpy()
    np.testing.assert_allclose(y.reshape(-1), np.array(expected, np.float64), rtol=1e-6, atol=1e-6)


def _center_scale_for_box(box, H, W, crop):
    """crop_image_from_xy (utils/general.py:181-191) builds boxes from (center, scale):  s = crop / scale,
    y1 = (cy - s // 2) / H,  y2 = y1 + s / H (same for x).  Inverts that for a SQUARE normalised box; returns None when the box
    is not expressible (non-square in pixels)."""
    y1, x1, y2, x2 = [float(v) for v in box]
    sy, sx = (y2 - y1) * H, (x2 - x1) * W
    if abs(sy - sx) > 1e-9 or sy == 0:
        return None
    s = sy
    cy, cx = y1 * H + np.floor(s / 2), x1 * W + np.floor(s / 2)
    return (cy, cx), crop / s


@pytest.mark.parametrize("case", [c for c in TF_CROP if c[5] == 0.0 and c[4][0] == c[4][1] and c[4][0] > 1],
                         ids=[c[0] for c in TF_CROP if c[5] == 0.0 and c[4][0] == c[4][1] and c[4][0] > 1])
def test_tf_crop_and_resize_vectors(ctx, case):
    """crop_and_resize_op_test.cc tables through crop_image_kernel (h3d_crop_image_from_xy): every box of TF's tests that the
    reference's (center, scale) parametrisation can express, incl. the flipped boxes (negative scale) and the box that
    reaches outside the image (extrapolation value 0 at the reference's call site)."""
    _, (H, W), data, boxes, (ch, cw), _, expected = case
    img = np.array(data, f32).reshape(1, H, W, 1)
    exp = np.array(expected, f32).reshape(len(boxes), ch, cw)
    done = 0
    for bi, box in enumerate(boxes):
        cs = _center_scale_for_box(box, H, W, ch)
        if cs is None:
            continue
        (cy, cx), scale = cs
        y = ctx.crop_image_from_xy(_cuda(img), _cuda(np.array([[cy, cx]], f32)), ch, _cuda(np.array([scale], f32))).cpu().numpy()
        np.testing.assert_allclose(y[0, :, :, 0], exp[bi], rtol=1e-6, atol=1e-6)
        done += 1
    assert done >= 1


def test_tf_max_pool_valid_vector(ctx):
    """pooling_ops_test.py _testMaxPoolValidPadding: 1..27 as [1,3,3,3], 2x2 / 2 VALID -> [13, 14, 15]."""
    y = ctx.max_pool(_cuda(_seq((1, 3, 3, 3)))).cpu().numpy()
    np.testing.assert_array_equal(y.reshape(-1), [13, 14, 15])

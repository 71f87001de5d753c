"""GPU parity of the wgmma implicit-GEMM convolution (operator entry h3d_conv2d_tc) against the fp64 oracle."""
import numpy as np
import pytest
import torch

from oracle import tf1_ops as T

pytestmark = pytest.mark.gpu
f32 = np.float32

# tolerance on outputs of unit scale: 3-pass split modes are fp32-grade, single-pass modes are 16-bit grade
TOL = {"bf16x3": 5e-5, "fp16x3": 2e-5, "fp16": 6e-3, "bf16": 5e-2, "fp16_f8c": 2e-4}

CASES = [  # B,H,W,Cin,Cout,k
    (1, 16, 8, 64, 64, 1),      # one exact tile, one K block: the smallest possible case
    (1, 16, 8, 64, 64, 3),      # halo / zero padding
    (2, 32, 32, 128, 128, 3),   # several tiles, BN = 128
    (3, 40, 40, 64, 256, 3),    # (8,8,2) tiles with a ragged batch, 2 N tiles
    (1, 24, 40, 192, 128, 7),   # 7x7, 3 channel chunks, partial tiles
    (2, 20, 12, 100, 72, 3),    # channel padding on both sides
    (1, 64, 64, 256, 512, 3),   # long K loop, pipeline wrap-around, many tiles per CTA
    (2, 20, 40, 64, 64, 3),     # 64 -> 64 (conv1_2 shape): ragged rows and columns, several tiles
    (3, 64, 64, 64, 64, 3),     # 64 -> 64: more tiles than CTAs
    (2, 24, 48, 64, 128, 3),    # 64 -> 128 (conv2_1)
    (4, 80, 80, 128, 256, 3),   # 200 pixel tiles x 2 N tiles of 128
    (1, 24, 16, 64, 64, 3),     # odd number of pixel tiles
    (2, 48, 32, 128, 128, 3),   # Cout = 128, 2 K blocks per tap
]


@pytest.fixture(scope="module")
def ctx():
    from hand3d_b200 import runtime
    return runtime.default_context()


@pytest.mark.parametrize("prec", ["bf16x3", "fp16x3", "fp16", "bf16", "fp16_f8c"])
@pytest.mark.parametrize("case", CASES)
def test_conv2d_tc_vs_oracle(ctx, case, prec):
    B, H, W, Cin, Cout, k = case
    rng = np.random.default_rng(11)
    x = rng.normal(size=(B, H, W, Cin)).astype(f32)
    w = (rng.normal(size=(k, k, Cin, Cout)) / np.sqrt(k * k * Cin)).astype(f32)
    b = rng.normal(size=Cout).astype(f32)
    y = ctx.conv2d_tc(torch.from_numpy(x).cuda(), w, b, leaky=True, precision=prec).cpu().numpy()
    ref = T.leaky_relu(T.conv2d_same(x, w, b, 1, np.float64))
    err = np.abs(y - ref).max()
    assert err < TOL[prec], "max abs err %.3e (tolerance %.1e)" % (err, TOL[prec])


STRIDED = [  # B,H,W,Cin,Cout: the stride-2 layers of the lifting pyramids (nets/ColorHandPose3DNetwork.py:255-258,291-294)
    (2, 32, 32, 32, 32),      # conv_pose_0_2: Cin / Cout padded 32 -> 64
    (3, 16, 16, 64, 64),      # conv_pose_1_2 / conv_vp_0_2 geometry
    (5, 8, 8, 128, 128),      # conv_pose_2_2: (8,8,2) tiles, ragged batch
    (2, 8, 8, 256, 256),      # conv_vp_2_2: 4 N tiles
    (1, 12, 20, 21, 40),      # odd channel counts, partial tiles
    (2, 32, 32, 64, 64),      # 64 -> 64 with the stride-2 epilogue
    (2, 32, 32, 128, 128),    # N = 128 tiles with the stride-2 epilogue
]


@pytest.mark.parametrize("prec", ["bf16x3", "fp16x3", "fp16"])
@pytest.mark.parametrize("case", STRIDED)
def test_conv2d_tc_stride2_vs_oracle(ctx, case, prec):
    """stride 2 'SAME' on an even-sized map (pads 0 before / 1 after) = the odd pixels of the stride-1 result."""
    B, H, W, Cin, Cout = case
    rng = np.random.default_rng(13)
    x = rng.normal(size=(B, H, W, Cin)).astype(f32)
    w = (rng.normal(size=(3, 3, Cin, Cout)) / np.sqrt(9 * Cin)).astype(f32)
    b = rng.normal(size=Cout).astype(f32)
    y = ctx.conv2d_tc(torch.from_numpy(x).cuda(), w, b, leaky=True, precision=prec, stride=2).cpu().numpy()
    ref = T.leaky_relu(T.conv2d_same(x, w, b, 2, np.float64))
    assert y.shape == ref.shape
    err = np.abs(y - ref).max()
    assert err < TOL[prec], "max abs err %.3e (tolerance %.1e)" % (err, TOL[prec])


def test_conv2d_tc_padded_planes_chain(ctx):
    """Cout = 32 feeding a second layer: the padding channels of the split planes must be exact zeros (they are the next K)."""
    rng = np.random.default_rng(14)
    x = rng.normal(size=(2, 16, 16, 21)).astype(f32)
    w1 = (rng.normal(size=(3, 3, 21, 32)) / np.sqrt(9 * 21)).astype(f32); b1 = rng.normal(size=32).astype(f32)
    y1 = ctx.conv2d_tc(torch.from_numpy(x).cuda(), w1, b1, leaky=True, precision="fp16x3")
    ref = T.leaky_relu(T.conv2d_same(x, w1, b1, 1, np.float64))
    assert np.abs(y1.cpu().numpy() - ref).max() < TOL["fp16x3"]


def test_conv2d_tc_identity_weights(ctx):
    """Delta kernel = identity: any layout / swizzle / descriptor mistake shows up as permuted channels or pixels."""
    B, H, W, C = 1, 16, 16, 64
    x = np.random.default_rng(12).normal(size=(B, H, W, C)).astype(f32)
    w = np.zeros((3, 3, C, C), f32)
    w[1, 1] = np.eye(C, dtype=f32)
    y = ctx.conv2d_tc(torch.from_numpy(x).cuda(), w, np.zeros(C, f32), leaky=False, precision="fp16x3").cpu().numpy()
    np.testing.assert_allclose(y, x, atol=1e-6)
    w2 = np.zeros((3, 3, C, C), f32)
    w2[0, 2] = np.eye(C, dtype=f32)         # tap (kh=0, kw=2): y[h,w] = x[h-1, w+1]
    y2 = ctx.conv2d_tc(torch.from_numpy(x).cuda(), w2, np.zeros(C, f32), leaky=False, precision="fp16x3").cpu().numpy()
    ref = np.zeros_like(x); ref[:, 1:, :-1] = x[:, :-1, 1:]
    np.testing.assert_allclose(y2, ref, atol=1e-6)

"""The wgmma convolution (conv_tc_kernel) and its weight gradient (conv_wgrad_tc_kernel) on every pixel tile their choosers can pick,
every kernel size and stride the entries accept, and the K-chunk fold at its boundaries.

The tile decides the TMA box, how the 128 (64) rows of a tile map to (w, h, image), and which rows are ragged or zero-filled, so each
table below holds at least one shape per candidate of choose_tile / wgrad_geometry; tests/test_conv_tile_coverage_cpu.py asks the
library (h3d_conv2d_tc_geometry, h3d_conv2d_wgrad_geometry) which tile each shape runs on and fails when a candidate drops out.

Three kinds of check.  fp64 parity with the bounds of test_gpu_tc_conv.py / test_gpu_conv_backward.py.  Exact canaries: small-integer
operands, whose products and partial sums are integers below 2^24 and exact in one bf16 plane, against the integer convolution with
assert-equal; the position code gives every (image, row, column) its own integers and every filter tap its own output channel, so a
row mapped to the wrong pixel, image or tap is a wrong integer at a known place.  Bit-for-bit identities: an image does not depend on
the batch it is in, stride 2 is the stride-1 result at the odd pixels, device-packed weights equal host-packed ones."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from oracle import tf1_grads as G
from oracle import tf1_ops as T

pytestmark = pytest.mark.gpu
f32, f64 = np.float32, np.float64

TOL = {"bf16x3": 5e-5, "fp16x3": 2e-5, "fp16": 6e-3, "bf16": 5e-2, "fp16_f8c": 2e-4}                      # test_gpu_tc_conv.TOL
BWD_TOL = {"bf16x3": {"dx": 5e-5, "dw": 1e-4, "db": 1e-4}, "bf16": {"dx": 5e-2, "dw": 5e-2, "db": 5e-2}}   # test_gpu_conv_backward.TOL
CANARY32 = 0x7FC0A5A5     # a NaN no convolution of finite operands produces
GUARD = 4096              # floats after the output that must keep the canary

# ---------------------------------------------------------------------------------------------------------------- shape tables
# (B, H, W, Cin, Cout, ksize, stride, exact_fit).  exact_fit marks the shapes whose B, H and W are all multiples of the tile; every
# other shape is ragged in at least one of them.  A multi-image tile (TB > 1) is only chosen for maps smaller than one tile, so those
# shapes have B = TB + 1: one full box of images and one box holding a single image.  Maps of more than 256 pixels with Cout % 128
# == 0 run N = 128 tiles, everything else N = 64 (the tile in the comment is TW x TH x TB).
FWD_SHAPES = [
    # N = 64, one shape per tile
    (1, 13, 25, 64, 64, 3, 1, False),      # 16x8x1
    (1, 25, 21, 128, 64, 5, 1, False),     # 8x16x1
    (1, 11, 63, 64, 64, 7, 1, False),      # 32x4x1
    (1, 63, 9, 192, 64, 3, 1, False),      # 4x32x1
    (1, 5, 257, 64, 64, 5, 1, False),      # 64x2x1
    (1, 1, 129, 128, 64, 7, 1, False),     # 128x1x1
    (3, 5, 5, 64, 64, 3, 1, False),        # 8x8x2
    (3, 1, 9, 192, 64, 5, 1, False),       # 16x4x2
    (3, 9, 1, 64, 64, 7, 1, False),        # 4x16x2
    (5, 3, 5, 128, 64, 3, 1, False),       # 8x4x4
    (5, 5, 1, 64, 64, 5, 1, False),        # 4x8x4
    (9, 3, 3, 192, 64, 7, 1, False),       # 4x4x8
    (9, 1, 5, 64, 64, 3, 1, False),        # 8x2x8
    (33, 1, 2, 128, 64, 1, 1, False),      # 2x2x32
    (129, 1, 1, 100, 40, 1, 1, False),     # 1x1x128, channel padding on both sides
    # N = 128, one shape per tile
    (1, 13, 25, 128, 128, 5, 1, False),    # 16x8x1
    (1, 25, 21, 64, 128, 3, 1, False),     # 8x16x1
    (1, 11, 63, 192, 128, 1, 1, False),    # 32x4x1
    (1, 63, 9, 64, 256, 5, 1, False),      # 4x32x1
    (1, 5, 257, 128, 128, 3, 1, False),    # 64x2x1
    (1, 1, 257, 64, 128, 5, 1, False),     # 128x1x1
    (7, 7, 37, 64, 128, 3, 1, False),      # 8x8x2
    (7, 19, 14, 64, 128, 1, 1, False),     # 16x4x2
    (7, 14, 19, 128, 128, 3, 1, False),    # 4x16x2
    (3, 17, 33, 64, 128, 3, 1, False),     # 8x4x4
    (3, 33, 17, 64, 256, 1, 1, False),     # 4x8x4
    (6, 17, 17, 64, 128, 3, 1, False),     # 4x4x8
    (6, 9, 33, 128, 128, 1, 1, False),     # 8x2x8
    (16, 257, 1, 64, 128, 3, 1, False),    # 2x2x32
    (129, 257, 1, 64, 128, 1, 1, False),   # 1x1x128
    # exact fits: the lifting pyramids' small maps and the FC-as-1x1 layers over batch rows
    (2, 8, 8, 128, 128, 3, 1, True),       # 8x8x2
    (8, 4, 4, 256, 256, 3, 1, True),       # 4x4x8
    (32, 2, 2, 64, 64, 3, 1, True),        # 2x2x32
    (128, 1, 1, 512, 512, 1, 1, True),     # 1x1x128
    (2, 32, 32, 64, 128, 5, 1, True),      # 16x8x1, 16 pixel tiles of N = 128
    # stride 2 (even H and W): ksize 3, 5 and 7, each on two tiles and with one, two and three 64-channel chunks
    (3, 6, 6, 64, 64, 3, 2, False),
    (1, 12, 20, 128, 128, 3, 2, False),
    (5, 4, 4, 128, 64, 5, 2, False),
    (1, 20, 12, 192, 128, 5, 2, False),
    (2, 2, 66, 64, 64, 7, 2, False),
    (3, 10, 18, 192, 128, 7, 2, False),
    (9, 2, 6, 21, 40, 5, 2, False),
]
# one shape per kernel instance <BN, PASSES> for the single-pass and the fp8-corrected modes: <64,1>, <128,1>, <64,4>
SINGLE_PASS = [((3, 5, 5, 64, 64, 3, 1), "bf16"), ((3, 5, 5, 64, 64, 3, 1), "fp16"), ((7, 7, 37, 64, 128, 3, 1), "bf16"),
               ((7, 7, 37, 64, 128, 3, 1), "fp16"), ((9, 3, 3, 192, 64, 7, 1), "fp16_f8c"), ((1, 25, 21, 64, 128, 3, 1), "fp16_f8c")]
# (B, H, W, Cin, Cout): 1x1 layers whose K-block count Cin / 64 sits at, one before and one past a fold of the tensor-core partial
# sum (9 blocks in the 3-pass modes, 27 in the single-pass ones)
FOLD_3PASS = [(2, 9, 13, 512, 64), (2, 9, 13, 576, 64), (2, 9, 13, 640, 64), (2, 9, 13, 1152, 64), (2, 9, 13, 1216, 64),
              (1, 13, 25, 640, 128), (1, 13, 25, 1216, 128)]
FOLD_1PASS = [(2, 9, 13, 1664, 64), (2, 9, 13, 1728, 64), (2, 9, 13, 1792, 64), (1, 13, 25, 1792, 128)]
# forced N tiles: a large map (N = 128 by default) and a small one (N = 64 by default)
BN_SHAPES = [(1, 25, 21, 64, 128, 3, 1), (3, 5, 5, 64, 128, 3, 1)]

# (B, H, W, Cin, Cout, ksize, stride, exact_fit): the weight gradient's 64-pixel boxes over the layer's INPUT map (at stride 2 dy is
# spread to the odd pixels of that map); BN = 128 where align_up(Cin, 64) % 128 == 0.  The data gradient of each shape runs
# conv_tc_kernel on (B, H, W) with the roles of Cin and Cout exchanged.
BWD_SHAPES = [
    (1, 13, 13, 64, 64, 3, 1, False),      # 8x8x1
    (1, 11, 25, 128, 64, 5, 1, False),     # 16x4x1
    (1, 25, 11, 64, 128, 3, 1, False),     # 4x16x1
    (1, 5, 129, 128, 128, 1, 1, False),    # 32x2x1
    (1, 129, 5, 64, 64, 3, 1, False),      # 2x32x1
    (1, 1, 65, 128, 64, 5, 1, False),      # 64x1x1
    (1, 65, 1, 64, 64, 3, 1, False),       # 1x64x1
    (3, 1, 5, 128, 128, 3, 1, False),      # 8x4x2
    (3, 5, 1, 64, 64, 7, 1, False),        # 4x8x2
    (5, 3, 3, 128, 64, 3, 1, False),       # 4x4x4
    (9, 1, 3, 64, 128, 5, 1, False),       # 4x2x8
    (9, 3, 1, 128, 128, 3, 1, False),      # 2x4x8
    (17, 1, 2, 64, 64, 1, 1, False),       # 2x2x16
    (65, 1, 1, 100, 40, 1, 1, False),      # 1x1x64
    (4, 4, 4, 256, 256, 3, 1, True),       # 4x4x4 exact (the lifting pyramids' 4x4 maps)
    (64, 1, 1, 512, 512, 1, 1, True),      # 1x1x64 exact (FC-as-1x1)
    (2, 12, 22, 64, 64, 3, 1, False),      # 8x8x1, 12 pixel blocks: as many splits as blocks
    (2, 41, 45, 64, 64, 3, 1, False),      # 8x8x1, 72 pixel blocks shared by fewer splits
    (2, 9, 7, 192, 512, 5, 1, False),      # 600 tiles: no split although there are several pixel blocks
    (2, 12, 20, 64, 64, 5, 2, False),      # stride 2
    (3, 6, 6, 128, 64, 5, 2, False),
    (1, 20, 12, 64, 128, 7, 2, False),
    (5, 4, 4, 192, 64, 7, 2, False),
    (2, 16, 16, 128, 128, 3, 2, True),
]
BWD_BF16 = [(1, 13, 13, 64, 64, 3, 1), (1, 11, 25, 128, 64, 5, 1), (3, 6, 6, 128, 64, 5, 2)]      # <64,1> and <128,1>


def _id(s):
    return "x".join(str(int(v)) for v in s)


# ---------------------------------------------------------------------------------------------------------------- helpers
@pytest.fixture(scope="module")
def ctx():
    from hand3d_b200 import runtime
    c = runtime.default_context()
    yield c
    torch.cuda.synchronize()
    c.check_errors()


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def conv_guarded(ctx, x, w, b, stride=1, leaky=False, prec="bf16x3"):
    """h3d_conv2d_tc_dev into a NaN-filled buffer with GUARD floats after the output: every output element must be written, nothing
    behind it."""
    from hand3d_b200 import _lib
    B, H, W, Cin = x.shape
    k, _, _, Cout = w.shape
    n = B * (H // stride) * (W // stride) * Cout
    buf = torch.empty(n + GUARD, dtype=torch.int32, device="cuda").fill_(CANARY32)
    xg, wg, bg = _cu(x), _cu(w), _cu(b)
    _lib.check(ctx.lib.h3d_conv2d_tc_dev(ctx.h, _ptr(xg), _ptr(wg), _ptr(bg), _ptr(buf), B, H, W, Cin, Cout, k, stride, int(leaky),
                                         _lib.PRECISIONS[prec], C.c_void_p(torch.cuda.current_stream().cuda_stream)), "h3d_conv2d_tc_dev")
    bits = buf.cpu().numpy().view(np.uint32)
    assert (bits[n:] == CANARY32).all(), "%d floats written behind the output" % int((bits[n:] != CANARY32).sum())
    assert not (bits[:n] == CANARY32).any(), "%d output elements never written" % int((bits[:n] == CANARY32).sum())
    return bits[:n].view(f32).reshape(B, H // stride, W // stride, Cout)


def assert_exact(got, want, what):
    want = np.asarray(want, f64)
    assert got.shape == want.shape
    bad = got.astype(f64) != want
    if bad.any():
        i = tuple(int(v[0]) for v in np.nonzero(bad))
        raise AssertionError("%s: %d of %d values differ, first at %s: got %r, want %r" % (what, int(bad.sum()), bad.size, i, got[i], want[i]))


@functools.lru_cache(maxsize=None)
def fwd_problem(B, H, W, Cin, Cout, k, stride):
    """Outputs of unit scale, which TOL is stated for: x ~ N(0, 1), w ~ N(0, 1 / K) and a small bias.  (The hi + lo planes the entry
    writes resolve an output of magnitude 4 to 8 to 3.05e-5 only; a bias ~ N(0, 1) puts 0.5 % of the outputs there and the largest
    map of the table then measured 5.06e-5 in bf16x3 against TOL's 5e-5, with no term of the sum wrong.)"""
    rng = np.random.default_rng(71)
    x = rng.normal(size=(B, H, W, Cin)).astype(f32)
    w = (rng.normal(size=(k, k, Cin, Cout)) / np.sqrt(k * k * Cin)).astype(f32)
    b = (0.1 * rng.normal(size=Cout)).astype(f32)
    return x, w, b, T.conv2d_same(x.astype(f64), w.astype(f64), b.astype(f64), stride, f64)


def int_problem(B, H, W, Cin, Cout, k, prec="bf16x3"):
    """Random operands in [-4, 4] x [-2, 2]: |partial sums| <= 8 k^2 Cin < 2^24, and the outputs fit the 16 bits of the hi + lo
    planes the entry writes.  Single-pass bf16 writes one 8-bit plane: there x is in [-2, 2] and every output channel has 56 non-zero
    weights spread over the whole of K, so |y| <= 4 x 56 + 8 < 256."""
    rng = np.random.default_rng(72)
    w = rng.integers(-2, 3, size=(k, k, Cin, Cout)).astype(f32)
    b = rng.integers(-8, 9, size=Cout).astype(f32)
    if prec == "bf16":
        K = k * k * Cin
        keep = np.zeros((K, Cout), bool)
        for co in range(Cout):
            keep[rng.choice(K, size=min(K, 56), replace=False), co] = True
        w *= keep.reshape(k, k, Cin, Cout)
        return rng.integers(-2, 3, size=(B, H, W, Cin)).astype(f32), w, b
    return rng.integers(-4, 5, size=(B, H, W, Cin)).astype(f32), w, b


def position_problem(B, H, W, Cin, Cout, k):
    """x[b,h,w,c] = (1 + pixel index) (c + 1) mod 251: integers exact in one bf16 plane, and two channels together tell every pixel of
    the batch from every other.  Output channel t < k^2 is the delta kernel at tap t reading input channel t mod Cin; the channels
    after them read the centre tap through a channel permutation."""
    idx = (1 + np.arange(B * H * W, dtype=np.int64)).reshape(B, H, W, 1)
    x = ((idx * (1 + np.arange(Cin, dtype=np.int64))) % 251).astype(f32)
    w = np.zeros((k, k, Cin, Cout), f32)
    for co in range(Cout):
        if co < k * k:
            w[co // k, co % k, co % Cin, co] = 1.0
        else:
            w[k // 2, k // 2, (5 * co + 3) % Cin, co] = 1.0
    return x, w, np.zeros(Cout, f32)


def int_reference(x, w, b, stride):
    return T.conv2d_same(x.astype(f64), w.astype(f64), b.astype(f64), stride, f64)


# ---------------------------------------------------------------------------------------------------------------- forward
@pytest.mark.parametrize("leaky", [False, True], ids=["linear", "leaky"])
@pytest.mark.parametrize("prec", ["bf16x3", "fp16x3"])
@pytest.mark.parametrize("shape", FWD_SHAPES, ids=_id)
def test_forward_vs_fp64(ctx, shape, prec, leaky):
    B, H, W, Cin, Cout, k, s, _ = shape
    x, w, b, ref = fwd_problem(*shape[:7])
    y = ctx.conv2d_tc_dev(_cu(x), _cu(w), _cu(b), stride=s, leaky=leaky, precision=prec).cpu().numpy()
    ref = T.leaky_relu(ref) if leaky else ref
    assert y.shape == ref.shape
    err = np.abs(y - ref).max()
    assert err < TOL[prec], "max abs err %.3e (tolerance %.1e)" % (err, TOL[prec])


@pytest.mark.parametrize("shape,prec", SINGLE_PASS, ids=lambda v: v if isinstance(v, str) else _id(v))
def test_forward_single_pass_vs_fp64(ctx, shape, prec):
    x, w, b, ref = fwd_problem(*shape)
    y = ctx.conv2d_tc(_cu(x), w, b, leaky=True, precision=prec, stride=shape[6]).cpu().numpy()
    err = np.abs(y - T.leaky_relu(ref)).max()
    assert err < TOL[prec], "max abs err %.3e (tolerance %.1e)" % (err, TOL[prec])


@pytest.mark.parametrize("kind", ["integer", "position"])
@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
@pytest.mark.parametrize("shape", FWD_SHAPES, ids=_id)
def test_forward_exact_canary(ctx, shape, prec, kind):
    B, H, W, Cin, Cout, k, s, _ = shape
    x, w, b = int_problem(B, H, W, Cin, Cout, k, prec) if kind == "integer" else position_problem(B, H, W, Cin, Cout, k)
    y = conv_guarded(ctx, x, w, b, stride=s, leaky=False, prec=prec)
    assert_exact(y, int_reference(x, w, b, s), "y[b,h,w,co] of %s" % _id(shape))


@pytest.mark.parametrize("prec", ["bf16x3", "fp16x3"])
@pytest.mark.parametrize("shape", [s for s in FWD_SHAPES if s[0] > 1], ids=_id)
def test_forward_image_does_not_depend_on_the_batch(ctx, shape, prec):
    """The N tile is chosen from the layer geometry alone, so a single-image call runs the same arithmetic on another pixel tile: the
    first image, the last of the first box, the first of the second box and the last image must not change by a bit."""
    from hand3d_b200 import runtime
    B, H, W, Cin, Cout, k, s, _ = shape
    x, w, b, _ = fwd_problem(*shape[:7])
    pool = 2 if s == 2 else 0
    TB = runtime.conv2d_tc_geometry(B, H, W, Cout, pool, prec)[2]
    assert runtime.conv2d_tc_geometry(B, H, W, Cout, pool, prec)[3] == runtime.conv2d_tc_geometry(1, H, W, Cout, pool, prec)[3]
    xg, wg, bg = _cu(x), _cu(w), _cu(b)
    y = ctx.conv2d_tc_dev(xg, wg, bg, stride=s, leaky=True, precision=prec)
    for i in sorted({0, min(TB, B) - 1, min(TB, B - 1), B - 1}):
        y1 = ctx.conv2d_tc_dev(xg[i:i + 1].contiguous(), wg, bg, stride=s, leaky=True, precision=prec)
        assert torch.equal(y1[0], y[i]), "image %d of %d (TB = %d)" % (i, B, TB)


@pytest.mark.parametrize("prec", ["bf16x3", "fp16x3", "fp16"])
@pytest.mark.parametrize("shape", [s for s in FWD_SHAPES if s[6] == 2], ids=_id)
def test_stride2_is_the_stride1_result_at_the_odd_pixels(ctx, shape, prec):
    """TF 'SAME' at stride 2 on an even size pads (k - 1) / 2 - 1 before: for ksize 3, 5 and 7 alike output (i, j) is the stride-1
    output at (2 i + 1, 2 j + 1).  Both run the same tile, so the identity holds bit for bit."""
    x, w, b, _ = fwd_problem(*shape[:7])
    xg, wg, bg = _cu(x), _cu(w), _cu(b)
    y2 = ctx.conv2d_tc_dev(xg, wg, bg, stride=2, leaky=True, precision=prec)
    y1 = ctx.conv2d_tc_dev(xg, wg, bg, stride=1, leaky=True, precision=prec)
    assert torch.equal(y2, y1[:, 1::2, 1::2].contiguous())


def _fold_check(ctx, case, prec, exact=True):
    B, H, W, Cin, Cout = case
    x, w, b, ref = fwd_problem(B, H, W, Cin, Cout, 1, 1)
    y = ctx.conv2d_tc_dev(_cu(x), _cu(w), _cu(b), leaky=True, precision=prec).cpu().numpy()
    err = np.abs(y - T.leaky_relu(ref)).max()
    assert err < TOL[prec], "max abs err %.3e (tolerance %.1e)" % (err, TOL[prec])
    if exact:
        xi, wi, bi = int_problem(B, H, W, Cin, Cout, 1, prec)
        assert_exact(conv_guarded(ctx, xi, wi, bi, prec=prec), int_reference(xi, wi, bi, 1), "%d K blocks" % (Cin // 64))


@pytest.mark.parametrize("prec", ["bf16x3", "fp16x3"])
@pytest.mark.parametrize("case", FOLD_3PASS, ids=_id)
def test_fold_boundaries_three_pass(ctx, case, prec):
    _fold_check(ctx, case, prec)


@pytest.mark.parametrize("prec", ["bf16", "fp16"])
@pytest.mark.parametrize("case", FOLD_1PASS, ids=_id)
def test_fold_boundaries_single_pass(ctx, case, prec):
    _fold_check(ctx, case, prec, exact=prec == "bf16")     # the exact canary is stated for bf16 planes


@pytest.mark.parametrize("chunk", [1, 4, 9, 27])
def test_fold_length_tuning(ctx, chunk):
    """27 K blocks (3x3, 192 channels) folded every 1, 4 (a last, partial chunk of 3), 9 and 27 blocks: integers stay exact whatever
    the fold length, floats stay inside the tolerance."""
    shape = (2, 9, 13, 192, 64, 3, 1)
    x, w, b, ref = fwd_problem(*shape)
    try:
        ctx.set_tuning("tc_chunk_kb", chunk)
        for prec in ("bf16x3", "bf16"):
            xi, wi, bi = int_problem(*shape[:6], prec)
            y = ctx.conv2d_tc_dev(_cu(x), _cu(w), _cu(b), leaky=True, precision=prec).cpu().numpy()
            err = np.abs(y - T.leaky_relu(ref)).max()
            assert err < TOL[prec], "%s: max abs err %.3e (tolerance %.1e)" % (prec, err, TOL[prec])
            assert_exact(conv_guarded(ctx, xi, wi, bi, prec=prec), int_reference(xi, wi, bi, 1), "%s, fold every %d" % (prec, chunk))
    finally:
        ctx.set_tuning("tc_chunk_kb", 0)


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("shape", BN_SHAPES, ids=_id)
def test_forced_n_tile(ctx, shape, bn):
    from hand3d_b200 import runtime
    B, H, W, Cin, Cout, k, s = shape
    x, w, b, ref = fwd_problem(*shape)
    try:
        ctx.set_tuning("tc_bn", bn)
        assert runtime.conv2d_tc_geometry(B, H, W, Cout)[3] == bn
        for prec in ("bf16x3", "fp16x3", "bf16"):
            y = ctx.conv2d_tc_dev(_cu(x), _cu(w), _cu(b), leaky=True, precision=prec).cpu().numpy()
            err = np.abs(y - T.leaky_relu(ref)).max()
            assert err < TOL[prec], "%s: max abs err %.3e (tolerance %.1e)" % (prec, err, TOL[prec])
        for kind in (int_problem, position_problem):
            xi, wi, bi = kind(*shape[:6])
            assert_exact(conv_guarded(ctx, xi, wi, bi), int_reference(xi, wi, bi, 1), "BN = %d" % bn)
    finally:
        ctx.set_tuning("tc_bn", 0)


@pytest.mark.parametrize("prec", ["bf16x3", "fp16x3", "fp16", "bf16"])
@pytest.mark.parametrize("shape", [(1, 25, 21, 128, 64, 5, 1), (2, 12, 20, 100, 72, 5, 1), (5, 4, 4, 128, 64, 5, 2)], ids=_id)
def test_device_packed_weights_match_host_packed_ksize5(ctx, shape, prec):
    """The device packer's K order over 25 taps is the host packer's."""
    x, w, b, _ = fwd_problem(*shape)
    s = shape[6]
    packed = ctx.pack_conv(w, b, precision=prec)
    y_packed = ctx.conv2d_tc_packed(_cu(x), packed, leaky=True, stride=s)
    y_dev = ctx.conv2d_tc_dev(_cu(x), _cu(w), _cu(b), stride=s, leaky=True, precision=prec)
    assert torch.equal(y_dev, y_packed)


# ---------------------------------------------------------------------------------------------------------------- backward
def _err(g, ref):
    return float(np.abs(np.asarray(g, f64) - ref).max() / max(np.abs(ref).max(), 1e-30))


@functools.lru_cache(maxsize=None)
def bwd_problem(B, H, W, Cin, Cout, k, s):
    rng = np.random.default_rng(73)
    x = rng.normal(size=(B, H, W, Cin)).astype(f32)
    w = (rng.normal(size=(k, k, Cin, Cout)) / np.sqrt(k * k * Cin)).astype(f32)
    b = rng.normal(size=Cout).astype(f32) * 0.1
    dy = rng.normal(size=(B, H // s, W // s, Cout)).astype(f32)
    return x, w, b, dy


def _backward_vs_oracle(ctx, shape, prec):
    B, H, W, Cin, Cout, k, s = shape
    x, w, b, dy = bwd_problem(*shape)
    xg, wg, bg, dyg = _cu(x), _cu(w), _cu(b), _cu(dy)
    y = ctx.conv2d_tc_dev(xg, wg, bg, stride=s, leaky=True, precision=prec)
    got = ctx.conv2d_tc_backward(xg, y, dyg, wg, stride=s, leaky=True, precision=prec)
    again = ctx.conv2d_tc_backward(xg, y, dyg, wg, stride=s, leaky=True, precision=prec)
    for name, u, v in zip(("dx", "dw", "db"), got, again):
        assert torch.equal(u, v), "%s differs between two runs" % name
    ref = G.conv_grads(x, w, b, dy, s, leaky=True, pre=y.cpu().numpy())
    for name, g, r in zip(("dx", "dw", "db"), got, ref):
        e = _err(g.cpu().numpy(), r)
        assert e < BWD_TOL[prec][name], "%s normwise error %.3e (bound %.1e)" % (name, e, BWD_TOL[prec][name])


@pytest.mark.parametrize("shape", BWD_SHAPES, ids=_id)
def test_backward_vs_fp64(ctx, shape):
    _backward_vs_oracle(ctx, shape[:7], "bf16x3")


@pytest.mark.parametrize("shape", BWD_BF16, ids=_id)
def test_backward_single_pass_vs_fp64(ctx, shape):
    _backward_vs_oracle(ctx, shape, "bf16")


@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
@pytest.mark.parametrize("shape", BWD_SHAPES, ids=_id)
def test_backward_exact_canary(ctx, shape, prec):
    """Integer x and dy in [-4, 4] (|sums| <= 16 B H W < 2^24) and a kernel that gives input channel ci the delta at tap ci mod k^2
    into output channel perm[ci]: dx is dy shifted by the tap and permuted, dW the integer correlation of x and dy, db the column
    sums of dy, all exact."""
    B, H, W, Cin, Cout, k, s, _ = shape
    rng = np.random.default_rng(74)
    x = rng.integers(-4, 5, size=(B, H, W, Cin)).astype(f32)
    dy = rng.integers(-4, 5, size=(B, H // s, W // s, Cout)).astype(f32)
    perm = rng.permutation(max(Cin, Cout))
    w = np.zeros((k, k, Cin, Cout), f32)
    for ci in range(Cin):
        t = ci % (k * k)
        w[t // k, t % k, ci, perm[ci] % Cout] = 1.0
    dx, dw, db = ctx.conv2d_tc_backward(_cu(x), None, _cu(dy), _cu(w), stride=s, leaky=False, precision=prec)
    assert_exact(dx.cpu().numpy(), G.conv2d_backprop_input(dy, w, x.shape, s), "dx[b,h,w,ci]")
    assert_exact(dw.cpu().numpy(), G.conv2d_backprop_filter(x, dy, k, s), "dw[kh,kw,ci,co]")
    assert_exact(db.cpu().numpy(), G.bias_add_grad(dy), "db[co]")


@pytest.mark.parametrize("shape", BWD_SHAPES, ids=_id)
def test_weight_gradient_one_hot_dy(ctx, shape):
    """dy one-hot at the last pixel of the last image (the ragged corner of the last box), then at the first pixel of the first:
    dW[kh, kw, :, co0] is 3 x the x patch around that pixel, every other column of dW is zero."""
    B, H, W, Cin, Cout, k, s, _ = shape
    idx = (1 + np.arange(B * H * W, dtype=np.int64)).reshape(B, H, W, 1)
    x = ((idx * (1 + np.arange(Cin, dtype=np.int64))) % 251).astype(f32)       # the position code of the forward canary
    wz = torch.zeros((k, k, Cin, Cout), device="cuda")                          # only its shape is read without dx
    for (b0, h0, w0, co0) in ((B - 1, H // s - 1, W // s - 1, Cout - 1), (0, 0, 0, Cout // 2)):
        dy = np.zeros((B, H // s, W // s, Cout), f32)
        dy[b0, h0, w0, co0] = 3.0
        for prec in ("bf16x3", "bf16"):
            _, dw, db = ctx.conv2d_tc_backward(_cu(x), None, _cu(dy), wz, stride=s, leaky=False, precision=prec, need_dx=False)
            assert_exact(dw.cpu().numpy(), G.conv2d_backprop_filter(x, dy, k, s), "%s dw[kh,kw,ci,co], dy at %s" % (prec, (b0, h0, w0, co0)))
            assert db.cpu().numpy()[co0] == 3.0 and np.count_nonzero(db.cpu().numpy()) == 1


@pytest.mark.parametrize("shape", [s for s in BWD_SHAPES if s[0] % 2 == 0 and s[0] * s[1] * s[2] > 128], ids=_id)
def test_weight_gradient_equals_the_sum_over_half_batches(ctx, shape):
    """The split-K ranges partition the pixel blocks: a dropped or doubled block is an O(1) difference, the order of the fp32 sums
    one of 1e-7."""
    from hand3d_b200 import runtime
    B, H, W, Cin, Cout, k, s, _ = shape
    assert runtime.conv2d_wgrad_geometry(B, H, W, k, Cin, Cout)[5] > 1
    x, w, b, dy = bwd_problem(*shape[:7])
    xg, dyg, wg = _cu(x), _cu(dy), _cu(w)
    run = lambda lo, hi: ctx.conv2d_tc_backward(xg[lo:hi].contiguous(), None, dyg[lo:hi].contiguous(), wg, stride=s, leaky=False,  # noqa: E731
                                                need_dx=False)[1].cpu().numpy().astype(f64)
    whole, halves = run(0, B), run(0, B // 2) + run(B // 2, B)
    e = _err(whole, halves)
    assert e < 1e-6, "dW of the batch differs from the sum over its halves by %.3e (normwise)" % e

"""The convolution layer paths the stage builders use and the operator tests do not reach, one layer at a time through
h3d_conv2d_layer_planes (Context.conv_layer): the fused 2x2 max-pool over every pool-legal tile shape, plane and fp32 outputs at
channel offsets, PoseNet2D's permuted 192-channel concat input, the fp16_f8c planes, the two first-layer kernels, the unfused split
max-pool, and the descriptor refusals.

Every plane is checked bit for bit against tests/planes_oracle.py's encoding of the fp32 output of the same call (both come from one
set of epilogue registers), padding channels must be exact zeros and every byte outside the layer's channels keeps its canary.
Values are scale-relative as in test_gpu_tc_range.py: |y - ref| <= BOUND S with S = conv(|x|, |w|) + |b| (fp64), max-pooled alongside y
where the layer pools; decoded planes may add their format's resolution (planes_oracle.FORMAT_REL / FORMAT_ABS)."""
import os
import re
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import planes_oracle as P  # noqa: E402
from test_gpu_tc_range import BOUND  # noqa: E402
from hand3d_b200 import weights as Wt  # noqa: E402
from hand3d_b200.runtime import Context  # noqa: E402
from oracle import tf1_ops as T  # noqa: E402

pytestmark = pytest.mark.gpu
f32, f64 = np.float32, np.float64
MODES = ["bf16x3", "fp16x3", "fp16_f8c", "fp16", "bf16"]
PLANE_KEYS = ("hi", "lo", "l8", "h8")
CANARY = {"hi": Context.CANARY16, "lo": Context.CANARY16, "l8": Context.CANARY8, "h8": Context.CANARY8}


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _np(t):
    if t is None:
        return None
    a = t.cpu().numpy()
    return a.view(np.uint16) if a.dtype == np.int16 else a


def _pad64(c):
    return -(-c // 64) * 64


@pytest.fixture(scope="module")
def ctx():
    from hand3d_b200 import runtime
    return runtime.default_context()


def problem(B, H, W, Cin, Cout, k, seed, Cx=None):
    """x ~ N(0, 1) [B,H,W,Cx] (channels past Cin zero), w ~ N(0, 1/K), b ~ N(0, 1)."""
    rng = np.random.default_rng(seed)
    x = np.zeros((B, H, W, Cx or Cin), f32)
    x[..., :Cin] = rng.normal(size=(B, H, W, Cin))
    w = (rng.normal(size=(k, k, Cin, Cout)) / np.sqrt(k * k * Cin)).astype(f32)
    b = rng.normal(size=Cout).astype(f32)
    return x, w, b


def reference(x, w, b, leaky, pool):
    """fp64 act(conv) and its scale S, both max-pooled 2x2 when the layer pools."""
    Cin = w.shape[2]
    xs = np.asarray(x[..., :Cin], f64)
    ref = T.conv2d_same(xs, w.astype(f64), b.astype(f64), 1, f64)
    S = T.conv2d_same(np.abs(xs), np.abs(w.astype(f64)), np.abs(b.astype(f64)), 1, f64)
    if leaky:
        ref = T.leaky_relu(ref)
    if pool == 1:
        ref, S = T.max_pool_2x2(ref), T.max_pool_2x2(S)
    return ref, S


def check_layer(o, prec, Cout, ref, S, cy_off=0, cyf_off=0, bound=None, plane_init=None, pad_zero=True):
    """Canaries, zero padding, bit-exact planes (when yf was requested too) and values.  plane_init: the plane contents expected
    outside the layer's channels when the buffers were pre-filled (else the canaries).  Returns the planes of the layer's channels."""
    bound = BOUND[prec] if bound is None else bound
    Cout_pad = _pad64(Cout) if pad_zero else Cout
    used = P.PLANES[prec]
    got = {}
    if o["hi"] is not None:
        for key in PLANE_KEYS:
            a = _np(o[key])
            if key not in used:
                assert (a == CANARY[key]).all(), "%s: the %s plane was written" % (prec, key)
                continue
            outside = np.concatenate([a[..., :cy_off], a[..., cy_off + Cout_pad:]], -1)
            want = CANARY[key] if plane_init is None else np.concatenate(
                [plane_init[key][..., :cy_off], plane_init[key][..., cy_off + Cout_pad:]], -1)
            assert (outside == want).all(), "%s: %s plane written outside channels [%d, %d)" % (prec, key, cy_off, cy_off + Cout_pad)
            assert (a[..., cy_off + Cout:cy_off + Cout_pad] == 0).all(), "%s: %s padding channels are not zero" % (prec, key)
            got[key] = a[..., cy_off:cy_off + Cout]
    yf = None
    if o["yf"] is not None:
        a = _np(o["yf"])
        bits = a.view(np.uint32)
        outside = np.concatenate([bits[..., :cyf_off], bits[..., cyf_off + Cout:]], -1)
        assert (outside == Context.CANARY32).all(), "%s: fp32 output written outside channels [%d, %d)" % (prec, cyf_off, cyf_off + Cout)
        yf = a[..., cyf_off:cyf_off + Cout]
        e = float((np.abs(yf.astype(f64) - ref) / S).max())
        assert e < bound, "%s: fp32 output scale-relative error %.3e, bound %.1e" % (prec, e, bound)
        if got:
            want = P.encode(yf, prec)
            for key in used:
                bad = got[key] != want[key]
                assert not bad.any(), "%s: %d %s plane values differ from the encoding of the fp32 output, first at %s" % (
                    prec, int(bad.sum()), key, tuple(int(i[0]) for i in np.nonzero(bad)))
    if got:
        dec = P.decode(got, prec)
        lim = bound * S + P.FORMAT_REL[prec] * np.abs(ref) + P.FORMAT_ABS[prec]
        e = float((np.abs(dec - ref) / lim).max())
        assert e <= 1.0, "%s: decoded planes exceed the bound by a factor %.3f" % (prec, e)
    return got, yf


def run_and_check(ctx, prec, shape, Cin, Cout, k, pool, seed, leaky=True, **kw):
    B, H, W = shape
    x, w, b = problem(B, H, W, Cin, Cout, k, seed)
    o = ctx.conv_layer(_cu(x), w, b, prec, pool=pool, leaky=leaky, yf=True, **kw)
    ref, S = reference(x, w, b, leaky, pool)
    return check_layer(o, prec, Cout, ref, S, cy_off=kw.get("cy_off", 0), cyf_off=kw.get("cyf_off", 0))


# ------------------------------------------------------------------------------------------ fused max-pool over every tile shape
# choose_tile (conv_wgmma.cu) restated: the candidates in order, the pool filter (2x2 windows inside one warp), fewest tiles first
CANDIDATES = [(16, 8, 1), (8, 16, 1), (32, 4, 1), (4, 32, 1), (64, 2, 1), (128, 1, 1), (8, 8, 2), (16, 4, 2), (4, 16, 2), (8, 4, 4),
              (4, 8, 4), (4, 4, 8), (8, 2, 8), (2, 2, 32), (1, 1, 128)]
POOL_LEGAL = [c for c in CANDIDATES if c[0] % 2 == 0 and c[0] <= 16 and c[1] % 2 == 0]
TILE_SHAPES = {(16, 8, 1): (1, 2, 2), (8, 16, 1): (1, 10, 2), (4, 32, 1): (1, 18, 2), (8, 8, 2): (2, 2, 2), (16, 4, 2): (2, 2, 10),
               (4, 16, 2): (2, 10, 2), (8, 4, 4): (3, 2, 2), (4, 8, 4): (3, 6, 2), (4, 4, 8): (5, 2, 2), (8, 2, 8): (5, 2, 6),
               (2, 2, 32): (9, 2, 2)}


def choose_tile(B, H, W, pool):
    best, pick = None, None
    for c in CANDIDATES:
        if pool and c not in POOL_LEGAL:
            continue
        tiles = -(-W // c[0]) * -(-H // c[1]) * -(-B // c[2])
        if best is None or tiles < best:
            best, pick = tiles, c
    return pick


def test_tile_shapes_reach_every_pool_legal_candidate():
    assert len(POOL_LEGAL) == 11
    assert {choose_tile(*s, True): s for s in TILE_SHAPES.values()}.keys() == set(POOL_LEGAL)
    for tile, shape in TILE_SHAPES.items():
        assert choose_tile(*shape, True) == tile, (tile, shape)


@pytest.mark.parametrize("tile", list(TILE_SHAPES), ids=["%dx%dx%d" % t for t in TILE_SHAPES])
@pytest.mark.parametrize("prec", MODES)
def test_fused_pool_every_tile(ctx, prec, tile):
    """pool = 1 (conv1_2 / conv2_2 / conv3_4) on a map that selects one pool-legal tile: TB > 1 tiles leave their last images
    ragged, TW from 2 to 16 moves the vertical pooling partner (lane ^ TW) across the warp."""
    run_and_check(ctx, prec, TILE_SHAPES[tile], 64, 64, 3, 1, seed=60)


@pytest.mark.parametrize("geom", [((2, 160, 160), 64, 64), ((2, 80, 80), 128, 128), ((2, 40, 40), 256, 256)],
                         ids=["conv1_2", "conv2_2", "conv3_4"])
@pytest.mark.parametrize("prec", MODES)
def test_fused_pool_network_geometry(ctx, prec, geom):
    """The three pooled trunk layers at a 320x320 input's sizes: N = 128 tiles for 128 / 256 channels, and 400, 200 and 50 pixel
    tiles per N tile, so most CTAs of the 132-SM grid loop over several tiles."""
    shape, Cin, Cout = geom
    run_and_check(ctx, prec, shape, Cin, Cout, 3, 1, seed=61)


@pytest.mark.parametrize("prec", MODES)
def test_fused_pool_ties_and_negative_windows(ctx, prec):
    """Equal maxima: a 1x1 layer on a map constant over each 2x2 window gives four bit-identical values per window.  All-negative
    windows: channels with bias -40 stay negative after the leaky ReLU, whose maximum is 0.01 x the least negative sum."""
    rng = np.random.default_rng(62)
    B, H, W, Cin, Cout = 2, 12, 20, 128, 128
    xs = rng.normal(size=(B, H // 2, W // 2, Cin)).astype(f32)
    x = np.repeat(np.repeat(xs, 2, axis=1), 2, axis=2)
    x[1, :, 8:] = rng.normal(size=(H, W - 8, Cin))              # and windows without ties
    w = (rng.normal(size=(1, 1, Cin, Cout)) / np.sqrt(Cin)).astype(f32)
    b = rng.normal(size=Cout).astype(f32)
    b[::2] = -40.0
    o = ctx.conv_layer(_cu(x), w, b, prec, pool=1, yf=True)
    ref, S = reference(x, w, b, True, 1)
    _, yf = check_layer(o, prec, Cout, ref, S)
    assert (yf[..., ::2] < 0).all() and (yf[..., 1::2] > 0).any()


# ------------------------------------------------------------------------------------------ outputs at channel offsets
@pytest.mark.parametrize("pool", [0, 1])
@pytest.mark.parametrize("prec", MODES)
def test_planes_and_fp32_at_offsets(ctx, prec, pool):
    """Planes at Cy_total 192 / cy_off 64 (16-channel aligned, as the fp16_f8c planes need) and fp32 at Cyf_total 136 / cyf_off 36 from
    the same call, with and without the fused pool."""
    run_and_check(ctx, prec, (2, 12, 20), 64, 64, 3, pool, seed=63, Cy_total=192, cy_off=64, Cyf_total=136, cyf_off=36)


@pytest.mark.parametrize("layout", [(2, 0), (7, 3)], ids=["stage", "offset"])
@pytest.mark.parametrize("prec", MODES)
def test_handsegnet_conv6_2_head(ctx, prec, layout):
    """conv6_2 (1x1, 512 -> 2, linear) writes fp32 only through the masked scalar tail: Cyf_total = 2 as in the stage, and at an odd
    offset inside a wider row, whose neighbours must keep their canaries."""
    Cyf_total, cyf_off = layout
    x, w, b = problem(2, 8, 12, 512, 2, 1, seed=64)
    o = ctx.conv_layer(_cu(x), w, b, prec, leaky=False, planes=False, yf=True, Cyf_total=Cyf_total, cyf_off=cyf_off)
    ref, S = reference(x, w, b, False, 0)
    check_layer(o, prec, 2, ref, S, cyf_off=cyf_off)


@pytest.mark.parametrize("prec", MODES)
def test_handsegnet_conv6_1_planes(ctx, prec):
    """conv6_1 (1x1, 128 -> 512, leaky) into 512-channel planes."""
    run_and_check(ctx, prec, (2, 8, 12), 128, 512, 1, 0, seed=65)


def posenet_perm():
    """build_posenet's weight permutation of the 192-channel concat planes (encoding 0..127 | score map 128..148 | zero)."""
    perm = np.full(192, -1, np.int32)
    perm[:128] = 21 + np.arange(128)
    perm[128:149] = np.arange(21)
    return perm


@pytest.mark.parametrize("prec", MODES)
def test_posenet_concat_chain(ctx, prec):
    """conv5_2 (1x1, 512 -> 21, linear) writes fp32 score maps and planes at Cy_total 192 / cy_off 128 into a buffer that already holds
    conv4_7's planes at 0..127; conv6_1 (7x7, 149 -> 128) then reads the concat through the permutation, against fp64 on the
    reference-order concat [score map | encoding]."""
    rng = np.random.default_rng(66)
    B, H, W = 2, 16, 24
    enc = rng.normal(size=(B, H, W, 128)).astype(f32)             # conv4_7's output
    pre = {"hi": np.full((B, H, W, 192), Context.CANARY16, np.uint16), "lo": np.full((B, H, W, 192), Context.CANARY16, np.uint16),
           "l8": np.full((B, H, W, 192), Context.CANARY8, np.uint8), "h8": np.full((B, H, W, 192), Context.CANARY8, np.uint8)}
    for key, v in P.encode(enc, prec).items():
        pre[key][..., :128] = v
    out = {key: _cu(v.view(np.int16) if v.dtype == np.uint16 else v) for key, v in pre.items()}
    x5, w5, b5 = problem(B, H, W, 512, 21, 1, seed=67)
    o = ctx.conv_layer(_cu(x5), w5, b5, prec, leaky=False, yf=True, Cy_total=192, cy_off=128, out=out)
    ref5, S5 = reference(x5, w5, b5, False, 0)
    planes5, sm = check_layer(o, prec, 21, ref5, S5, cy_off=128, plane_init=pre)
    # conv6_1: its fp32 input holds exactly the values whose planes conv5_2 and conv4_7 left in the buffer (the split on the device
    # reproduces them bit for bit: checked above for the score map, by construction for the encoding)
    xcat = np.zeros((B, H, W, 192), f32)
    xcat[..., :128] = enc
    xcat[..., 128:149] = sm
    for key, v in P.encode(xcat, prec).items():
        np.testing.assert_array_equal(v[..., :149], _np(o[key])[..., :149])
    w6 = (rng.normal(size=(7, 7, 149, 128)) / np.sqrt(49 * 149)).astype(f32)
    b6 = rng.normal(size=128).astype(f32)
    o6 = ctx.conv_layer(_cu(xcat), w6, b6, prec, perm=posenet_perm(), yf=True)
    ref6, S6 = reference(np.concatenate([sm, enc], -1), w6, b6, True, 0)
    check_layer(o6, prec, 128, ref6, S6)


# ------------------------------------------------------------------------------------------ first layer (route 1)
FIRST_SHAPES = [(2, 19, 45), (1, 8, 8), (3, 40, 24)]


def first_layer_problem(shape, seed):
    B, H, W = shape
    rng = np.random.default_rng(seed)
    x = Wt.synthetic_images(B, H, W, seed=seed)
    w = (rng.normal(size=(3, 3, 3, 64)) * np.sqrt(2.0 / 27)).astype(f32)
    b = (rng.normal(size=64) * 0.1).astype(f32)
    return x, w, b


@pytest.mark.parametrize("layout", [(64, 0), (128, 56)], ids=["stage", "offset"])
@pytest.mark.parametrize("shape", FIRST_SHAPES, ids=["x".join(map(str, s)) for s in FIRST_SHAPES])
@pytest.mark.parametrize("prec", ["bf16x3", "fp16x3", "fp16", "bf16"])
def test_first_layer_tc_kernel(ctx, prec, shape, layout):
    """conv1_1 on conv_c3_tc_kernel (planes only, the default): values, the split invariant of planes_oracle.split_ok, zero planes of
    the other formats and canaries around the channels."""
    Cy_total, cy_off = layout
    x, w, b = first_layer_problem(shape, seed=70)
    ctx.set_tuning("c3_ffma", 0)
    o = ctx.conv_layer(_cu(x), w, b, prec, route=1, Cy_total=Cy_total, cy_off=cy_off)
    ref, S = reference(x, w, b, True, 0)
    got, _ = check_layer(o, prec, 64, ref, S, cy_off=cy_off)
    if "lo" in got:
        ok = P.split_ok(got["hi"], got["lo"], P.HALF[prec])
        assert ok.all(), "%s: %d planes break the split invariant" % (prec, int((~ok).sum()))


@pytest.mark.parametrize("shape", FIRST_SHAPES, ids=["x".join(map(str, s)) for s in FIRST_SHAPES])
@pytest.mark.parametrize("prec", MODES)
def test_first_layer_ffma_kernel_planes(ctx, prec, shape):
    """conv1_1 on conv3x3_c3_kernel (the c3_ffma switch, and always in fp16_f8c) with yf requested: fp32-grade values and every
    plane the encoding of yf."""
    x, w, b = first_layer_problem(shape, seed=71)
    ctx.set_tuning("c3_ffma", 1)
    try:
        o = ctx.conv_layer(_cu(x), w, b, prec, route=1, yf=True, Cy_total=64)
    finally:
        ctx.set_tuning("c3_ffma", 0)
    ref, S = reference(x, w, b, True, 0)
    check_layer(o, prec, 64, ref, S, bound=BOUND["fp32"])


# ------------------------------------------------------------------------------------------ unfused split max-pool
@pytest.fixture(scope="module")
def stage_inputs(ctx):
    ctx.load_weights(Wt.synthetic_weights(0))
    return Wt.synthetic_images(2, 64, 96, seed=72), Wt.synthetic_images(1, 64, 64, seed=73)


def _stages(ctx, prec, img, crop, no_fusion):
    ctx.set_precision(prec)
    ctx.set_tuning("no_pool_fusion", int(no_fusion))
    try:
        return [ctx.handsegnet(_cu(img)).cpu()] + [s.cpu() for s in ctx.posenet(_cu(crop))]
    finally:
        ctx.set_tuning("no_pool_fusion", 0)
        ctx.set_precision("bf16x3")


@pytest.mark.parametrize("prec", ["bf16x3", "fp16x3", "fp16", "bf16"])
def test_unfused_pool_equals_fused(ctx, stage_inputs, prec):
    """no_pool_fusion: conv1_2 / conv2_2 / conv3_4 store their planes and maxpool_split_kernel pools them.  Both paths carry the
    arg-max element's value through the same split (the fused one pools the fp32 values and splits the maximum, the unfused one
    keeps the (hi, lo) pair of the largest hi + lo) and the convolution's per-pixel arithmetic does not depend on the tile shape, so
    HandSegNet and all three PoseNet2D score maps are bit-identical."""
    img, crop = stage_inputs
    fused = _stages(ctx, prec, img, crop, False)
    unfused = _stages(ctx, prec, img, crop, True)
    for i, (a, b) in enumerate(zip(fused, unfused)):
        assert torch.equal(a, b), "%s output %d: max |fused - unfused| = %.3e" % (prec, i, float((a - b).abs().max()))


def test_unfused_pool_refused_in_fp16_f8c(ctx, stage_inputs):
    img, _ = stage_inputs
    with pytest.raises(RuntimeError, match="code -1.*fp16_f8c: max-pool must be fused"):
        _stages(ctx, "fp16_f8c", img, img, True)


# ------------------------------------------------------------------------------------------ refusals
REFUSALS = [  # id, precision, (B, H, W), Cout, conv_layer arguments, message
    ("pool_cout21", "bf16x3", (1, 8, 8), 21, dict(pool=1), "fused pooling needs Cout % 32 == 0"),
    ("pool_odd_h", "bf16x3", (1, 9, 8), 64, dict(pool=1), "needs even H and W"),
    ("pool_odd_w", "fp16", (1, 8, 7), 64, dict(pool=1), "needs even H and W"),
    ("split_off4", "bf16x3", (1, 8, 8), 64, dict(Cy_total=128, cy_off=4), "split output channel offset/stride must be multiples of 8"),
    ("fp8_off8", "fp16_f8c", (1, 8, 8), 64, dict(Cy_total=128, cy_off=8), "fp8 planes need 16-channel aligned offsets"),
    ("fp32_off2", "bf16x3", (1, 8, 8), 64, dict(yf=True, Cyf_total=66, cyf_off=2), "fp32 output channel offset/stride must be multiples of 4"),
]


@pytest.mark.parametrize("prec,shape,Cout,kw,msg", [pytest.param(*r[1:], id=r[0]) for r in REFUSALS])
def test_descriptor_refusals(ctx, prec, shape, Cout, kw, msg):
    """Illegal layer descriptors come back as H3D_EINVAL (-1) with the descriptor's message, and nothing is written."""
    B, H, W = shape
    kw = dict(kw)
    x, w, b = problem(B, H, W, 64, Cout, 3, seed=74)
    Cy_total = kw.pop("Cy_total", _pad64(Cout))
    out = {key: torch.full((B, H, W, Cy_total), CANARY[key], dtype=torch.int16 if key in ("hi", "lo") else torch.uint8, device="cuda")
           for key in PLANE_KEYS}
    with pytest.raises(RuntimeError, match=r"\(code -1\): tc_conv: .*" + re.escape(msg)):
        ctx.conv_layer(_cu(x), w, b, prec, Cy_total=Cy_total, out=out, **kw)
    for key in PLANE_KEYS:
        assert (_np(out[key]) == CANARY[key]).all(), key

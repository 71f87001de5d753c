"""The resize, pooling, crop and key-point arg-max kernels of csrc/elementwise.cu on every path their launchers choose.

Each table row is marked with the kernel it must reach, restated here from the launchers' predicates (resize_kernel, maxpool_kernel,
crop_path, detect_grid, upsample_kernel); test_dispatch runs one row per kernel under torch.profiler and checks the names, and
tests/test_postprocess_coverage_cpu.py checks without a GPU that every __global__ of elementwise.cu is reached by some row or excluded
with a reason.

All comparisons are against the numpy restatements in oracle/tf1_ops.py and oracle/hand3d_oracle.py, or np.argmax: the resize, the
max-pool and the crop bit for bit, avgpool8 against an fp64 mean within the error bound of its 64-term fp32 sum (and exactly on
integer-valued inputs), the arg-max exactly.  The arg-max maps carry plateaus across thread, slot and CTA boundaries, maxima at the last
pixel, constant maps, +-inf, -0.0 / +0.0 ties in both orders and NaNs of both signs before and after the maximum: np.argmax ranks
-0.0 equal to +0.0 and every NaN above everything, first occurrence first.

Every run writes into buffers filled with a NaN canary and followed by guard words (test_gpu_conv_direct_paths.Guarded); every row
also checks that each image gives the same bits alone as inside its batch and that two runs give the same bits.  Shapes the kernels
cannot handle are refused by the operator entries with H3D_EINVAL and a message before anything is enqueued (test_*_refused)."""
import ctypes as C
import functools
import os
import re
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
for _p in (os.path.dirname(HERE), HERE):        # the repository (also when run as the dispatch child) and tests/
    if _p not in sys.path:
        sys.path.insert(0, _p)
from hand3d_b200 import _lib, runtime  # noqa: E402
from oracle import hand3d_oracle as O  # noqa: E402
from oracle import tf1_ops as T  # noqa: E402
from test_gpu_conv_direct_paths import Guarded  # noqa: E402

pytestmark = pytest.mark.gpu
f32, f64 = np.float32, np.float64
WAVE = 132 * 8                  # crop_image_kernel / seg_prob_kernel: about one resident wave of 256-thread CTAs, split over the images
MAX_GRID_IMAGES = 65535         # gridDim.y: the most images one call of the per-image-grid-row kernels takes
# avgpool8_kernel sums the 64 window values one after another in fp32 and divides by 64 (exact): |y - mean| <= gamma_63 sum|x| / 64,
# gamma_n = n u / (1 - n u), u = 2^-24 (Higham, Accuracy and Stability of Numerical Algorithms, (4.4))
GAMMA_63 = 63 * 2.0 ** -24 / (1 - 63 * 2.0 ** -24)


def _cd(a, b):
    return -(-a // b)


# ---------------------------------------------------------------------------------------------------------------- kernel choice
def resize_kernel(H, W, C, oh, ow):
    """launch_resize_bilinear_tf1"""
    if (H, W) == (oh, ow):
        return "copy"
    return "resize_bilinear_tf1_kernel<%d>" % (C if C in (21, 2) else 0)


def maxpool_kernel(C):
    return "maxpool_f32_kernel" if C % 4 == 0 else "maxpool_f32_scalar_kernel"


def crop_grid(B, crop):
    """launch_crop_image: CTAs per image"""
    return max(1, min(_cd(crop * crop, 256), _cd(WAVE, B)))


def crop_path(B, C, crop):
    path = ["c3" if C == 3 else "channels"]
    if crop == 1:
        path.append("single")
    if crop_grid(B, crop) * 256 < crop * crop:
        path.append("loop")
    return "+".join(path)


def detect_grid(H, W, C):
    """launch_detect_keypoints: (pixels per CTA step P, CTAs per image)"""
    P = max(1, 256 // C)
    return P, max(1, min(_cd(H * W, P * 16), 64))


def upsample_kernel(H, W, oh, ow, aligned=True):
    """launch_resize_argmax21"""
    s = oh // H
    if (oh % H == 0 and ow % W == 0 and oh // H == ow // W and s & (s - 1) == 0 and s >= 2 and ow % 4 == 0 and aligned
            and W * 21 * 8 + 4 * 16 * 21 * 8 <= 48 * 1024):
        return "resize_argmax_pow2_kernel"
    return "resize_argmax_kernel"


# ---------------------------------------------------------------------------------------------------------------- tables
# h3d_resize_bilinear_tf1: (B, H, W, C, out_h, out_w, kernel)
RESIZE = [
    (2, 32, 32, 21, 256, 256, "resize_bilinear_tf1_kernel<21>"),   # x8, float4 rows
    (4, 32, 32, 21, 256, 256, "resize_bilinear_tf1_kernel<21>"),   # more float4 groups than one grid: the grid-stride loop
    (1, 30, 40, 21, 45, 61, "resize_bilinear_tf1_kernel<21>"),     # non-integer up, rows of 1281 floats: scalar tail
    (2, 64, 48, 21, 17, 13, "resize_bilinear_tf1_kernel<21>"),     # non-integer down, tail
    (1, 5, 7, 21, 1, 13, "resize_bilinear_tf1_kernel<21>"),        # one output row
    (3, 40, 40, 2, 320, 320, "resize_bilinear_tf1_kernel<2>"),     # float4
    (2, 17, 23, 2, 5, 7, "resize_bilinear_tf1_kernel<2>"),         # down, tail
    (2, 16, 12, 2, 7, 12, "resize_bilinear_tf1_kernel<2>"),        # only H changes
    (1, 1, 9, 2, 4, 9, "resize_bilinear_tf1_kernel<2>"),           # one input row, only H changes, tail
    (1, 12, 10, 3, 30, 17, "resize_bilinear_tf1_kernel<0>"),       # tail
    (2, 48, 64, 5, 24, 32, "resize_bilinear_tf1_kernel<0>"),       # exact x1/2, float4
    (1, 1, 1, 4, 7, 9, "resize_bilinear_tf1_kernel<0>"),           # one input pixel
    (2, 9, 11, 1, 1, 1, "resize_bilinear_tf1_kernel<0>"),          # one output pixel
    (2, 16, 12, 3, 16, 29, "resize_bilinear_tf1_kernel<0>"),       # only W changes
    (2, 3, 1, 1, 1000, 1, "resize_bilinear_tf1_kernel<0>"),        # x333 in H alone
    (1, 8, 8, 21, 8, 8, "copy"),
    (3, 5, 3, 7, 5, 3, "copy"),
]

# h3d_maxpool2x2_f32: (B, H, W, C, kernel)
MAXPOOL = [
    (2, 16, 24, 64, "maxpool_f32_kernel"),
    (2, 17, 25, 8, "maxpool_f32_kernel"),                # odd H and W: VALID drops the last row and column
    (1, 2, 2, 4, "maxpool_f32_kernel"),
    (1, 3, 5, 4, "maxpool_f32_kernel"),
    (2, 258, 258, 256, "maxpool_f32_kernel"),            # grid-stride loop
    (2, 15, 9, 21, "maxpool_f32_scalar_kernel"),
    (3, 2, 3, 1, "maxpool_f32_scalar_kernel"),
    (1, 33, 2, 3, "maxpool_f32_scalar_kernel"),
    (2, 7, 6, 2, "maxpool_f32_scalar_kernel"),
    (2, 8, 6, 3, "maxpool_f32_scalar_kernel"),
    (3, 301, 299, 21, "maxpool_f32_scalar_kernel"),      # grid-stride loop
]

# h3d_avgpool8: (B, H, W, C)
AVGPOOL = [(1, 8, 8, 1), (2, 16, 24, 3), (1, 32, 8, 21), (3, 8, 40, 64), (2, 256, 256, 21)]

# h3d_crop_image_from_xy: (B, H, W, C, crop, boxes, path); boxes "random" (centres around and outside the image, scales 0.25 .. 20)
# or "edge" (samples exactly on rows / columns 0 and H-1 / W-1, and just outside them)
CROP = [
    (1, 320, 320, 3, 256, "random", "c3"),                   # one pass: 256 CTAs of 256 pixels
    (6, 240, 320, 3, 256, "random", "c3+loop"),              # 176 CTAs per image: the grid-stride loop
    (6, 60, 80, 1, 255, "random", "channels+loop"),
    (2, 37, 29, 2, 3, "random", "channels"),
    (3, 20, 30, 4, 2, "random", "channels"),
    (2, 50, 40, 21, 368, "random", "channels+loop"),
    (4, 1, 30, 3, 16, "random", "c3"),                       # one-pixel-high image
    (4, 25, 1, 2, 16, "random", "channels"),                 # one-pixel-wide image
    (2, 1, 1, 4, 5, "random", "channels"),
    (5, 30, 30, 3, 1, "random", "c3+single"),                # crop 1 samples the box centre
    (3, 30, 30, 21, 1, "random", "channels+single"),
    (1100, 6, 5, 1, 32, "random", "channels+loop"),          # one CTA per image
    (4, 41, 33, 3, 64, "edge", "c3"),
    (4, 41, 33, 4, 64, "edge", "channels"),
    (4, 23, 37, 1, 255, "edge", "channels"),
]
CROP_SCALES = [0.25, 1.0, 5.0, 7.5, 0.6, 2.048, 20.0]

# h3d_detect_keypoints: (B, H, W, C); C in {1, 2, 21, 64, 255, 256}, H W not a multiple of P, one to 64 CTAs per image
DETECT = [
    (14, 300, 301, 1),          # P = 256, 23 CTAs
    (14, 37, 41, 1),            # one CTA
    (7, 45, 47, 2),
    (2, 64, 61, 21),
    (1, 256, 251, 21),          # 64 CTAs, several steps per thread
    (1, 33, 35, 64),
    (1, 27, 29, 255),           # P = 1
    (1, 25, 41, 256),
]

# h3d_upsample_detect_keypoints: (B, H, W, out_h, out_w, aligned output, kernel)
UPSAMPLE = [
    (3, 32, 32, 256, 256, True, "resize_argmax_pow2_kernel"),     # the pipeline's x8
    (2, 30, 40, 240, 320, True, "resize_argmax_pow2_kernel"),
    (2, 16, 40, 32, 80, True, "resize_argmax_pow2_kernel"),       # x2
    (2, 9, 7, 72, 56, True, "resize_argmax_pow2_kernel"),
    (1, 4, 228, 16, 912, True, "resize_argmax_pow2_kernel"),      # the widest row the shared memory takes
    (2, 1, 1, 8, 8, True, "resize_argmax_pow2_kernel"),
    (1, 4, 229, 16, 916, True, "resize_argmax_kernel"),           # one column wider
    (1, 20, 12, 60, 36, True, "resize_argmax_kernel"),            # x3
    (2, 48, 48, 64, 64, True, "resize_argmax_kernel"),            # x4/3
    (2, 40, 36, 20, 18, True, "resize_argmax_kernel"),            # x1/2
    (2, 9, 7, 36, 14, True, "resize_argmax_kernel"),              # x4 and x2
    (2, 9, 5, 18, 10, True, "resize_argmax_kernel"),              # x2, out_w % 4 != 0
    (2, 16, 16, 128, 128, False, "resize_argmax_kernel"),         # output not 16-byte aligned
    (2, 1, 1, 3, 5, True, "resize_argmax_kernel"),
]

# h3d_seg_postprocess's max_loc (seg_prob_kernel): (B, H, W); fg plateaus across the CTAs of an image
SEG = [(2, 320, 320), (3, 100, 70), (1, 41, 500)]


def _id(s):
    return "x".join(str(v) for v in s)


def expected_kernels():
    """{kernel name: rows} over every table"""
    out = {}
    for r in RESIZE:
        out.setdefault(r[-1], []).append(r)
    for r in MAXPOOL:
        out.setdefault(r[-1], []).append(r)
    for r in AVGPOOL:
        out.setdefault("avgpool8_kernel", []).append(r)
    for r in CROP:
        out.setdefault("crop_image_kernel", []).append(r)
    for r in DETECT:
        out.setdefault("heatmap_argmax_kernel", []).append(r)
        out.setdefault("argmax_decode_kernel", []).append(r)
    for r in UPSAMPLE:
        out.setdefault(r[-1], []).append(r)
        out.setdefault("argmax_decode_kernel", []).append(r)
    for r in SEG:
        out.setdefault("seg_prob_kernel<false>", []).append(r)
    return out


# ---------------------------------------------------------------------------------------------------------------- arg-max maps
NAN_NEG = np.array([0xFFC00000], np.uint32).view(f32)[0]      # a NaN with the sign bit set
NAN_POS_PAYLOAD = np.array([0x7F800001], np.uint32).view(f32)[0]


def spots(n, P, gx, rng):
    """Two pixel indices a < b of a map of n pixels: where possible, a in the last CTA's first step and b in CTA 0's second step, so that
    the first occurrence is found by a later CTA; else two distinct random pixels."""
    a, b = P * (gx - 1) + P // 2, gx * P + P // 3
    if gx > 1 and b < n - 1:
        return a, b
    a, b = sorted(rng.choice(max(n - 1, 2), 2, replace=False)) if n > 2 else (0, n - 1)
    return int(a), int(b)


PATTERNS = ["random", "plateau", "run", "last", "const", "const_neg_zero", "inf", "all_neg_inf", "neg_zero_first", "pos_zero_first",
            "nan_neg_before", "nan_pos_after", "nan_both", "all_nan"]


def pattern_map(kind, n, P, gx, rng, cand=None):
    """A flat map of n pixels.  cand (optional): the pixels the special values may go to (for the up-sampling: input pixels that an
    output samples exactly, away from the last row and column)."""
    m = (rng.normal(size=n) * 0.5 - 3.0).astype(f32)
    pick = np.arange(n) if cand is None else np.asarray(cand)
    if pick.size < 2:
        pick = np.arange(n)
    a, b = spots(pick.size, P, gx, rng)
    a, b = int(pick[a]), int(pick[b])
    if kind == "random":
        return (rng.normal(size=n)).astype(f32)
    if kind == "plateau":       # the maximum at a, in the next thread, the next step of a's thread, another CTA, b and the last pixel
        for q in (a, a + 1, a + P, a + P * gx, a + 16 * P, b, n - 1):
            if q < n:
                m[q] = 2.0
        return m
    if kind == "run":           # one run of the maximum over three steps' worth of threads
        m[a:a + 3 * P] = 2.0
        return m
    if kind == "last":
        m[n - 1] = 2.0
        return m
    if kind == "const":
        return np.full(n, 0.75, f32)
    if kind == "const_neg_zero":
        return np.full(n, -0.0, f32)
    if kind == "inf":
        m[:] = -np.inf
        m[a] = m[b] = np.inf
        return m
    if kind == "all_neg_inf":
        return np.full(n, -np.inf, f32)
    if kind == "neg_zero_first":
        m[a], m[b] = -0.0, 0.0
        return m
    if kind == "pos_zero_first":
        m[a], m[b] = 0.0, -0.0
        return m
    if kind == "nan_neg_before":
        m[b] = 2.0
        m[a] = NAN_NEG
        return m
    if kind == "nan_pos_after":
        m[a] = 2.0
        m[b] = NAN_POS_PAYLOAD
        return m
    if kind == "nan_both":
        m[a], m[b] = NAN_NEG, np.nan
        m[n - 1] = 2.0
        return m
    if kind == "all_nan":
        return np.full(n, NAN_NEG, f32)
    raise ValueError(kind)


@functools.lru_cache(maxsize=None)
def detect_problem(B, H, W, C):
    """scoremaps [B,H,W,C] whose (image, channel) maps cycle through PATTERNS"""
    rng = np.random.default_rng(B * 1000003 + H * 1009 + W * 31 + C)
    P, gx = detect_grid(H, W, C)
    s = np.empty((B, H * W, C), f32)
    for b in range(B):
        for c in range(C):
            s[b, :, c] = pattern_map(PATTERNS[(b * C + c) % len(PATTERNS)], H * W, P, gx, rng)
    return s.reshape(B, H, W, C)


def argmax_uv(maps):
    """np.argmax per channel of [B,H,W,C] -> [B,C,2] (row, col) int32"""
    B, H, W, C = maps.shape
    idx = np.argmax(maps.reshape(B, H * W, C), axis=1)
    return np.stack([idx // W, idx % W], -1).astype(np.int32)


def exact_pixels(H, W, oh, ow):
    """Flat indices of the input pixels that some output pixel samples with weights (0, 0), on even rows and columns and not on the
    last row or column: a -0.0 there keeps its sign in the output only while its right and lower neighbours are negative"""
    iy = np.arange(oh, dtype=f32) * (f32(H) / f32(oh))
    ix = np.arange(ow, dtype=f32) * (f32(W) / f32(ow))
    ys = sorted({int(v) for v in iy if v == np.floor(v) and v < H - 1 and int(v) % 2 == 0})
    xs = sorted({int(v) for v in ix if v == np.floor(v) and v < W - 1 and int(v) % 2 == 0})
    return [y * W + x for y in ys for x in xs]


def thread_order_case(H, W, s):
    """The power-of-two kernel walks a thread's pixels row by row inside a column group, then the next group 16 groups (64 pixels) on.
    Input pixel (y0, xa) = 1 - 2^-24 and (y0 + 1, xa) = 1 make output rows s y0 + s/2 .. s y0 + s - 1 of column s xa round to 1; input
    pixel (y0, xb) = 1, xb = xa + 64 / s, makes output row s y0 of column s xb exactly 1, in the same thread and value slot.  The
    thread meets the maximum at row s y0 + s/2 first, np.argmax takes row s y0: the tie test inside the thread decides."""
    y0, xa = 0, 1
    xb = xa + 64 // s
    if s < 2 or xb >= W - 1 or H < 2:
        return None
    x = np.full((H, W), -3.0, f32)
    x[y0, xa], x[y0 + 1, xa], x[y0, xb] = f32(1.0) - f32(2.0 ** -24), 1.0, 1.0
    return x


def last_slot_case(H, W, s):
    """Input pixels (0, xa) = 1 - (s/2) 2^-24 and (0, xa + 1) = 1, xa = 64 / s - 1: the interpolants of output row 0 reach 1 first at
    column 63 (lx = (s-1)/s rounds up, (s-2)/s does not), the last of the power-of-two kernel's 64 value slots of a channel
    (column group 15, pixel offset 3)."""
    xa = 64 // s - 1
    if s < 2 or xa + 1 > W - 1 or H < 2:
        return None
    x = np.full((H, W), -3.0, f32)
    x[0, xa], x[0, xa + 1] = f32(1.0) - f32(s / 2 * 2.0 ** -24), 1.0
    return x


@functools.lru_cache(maxsize=None)
def upsample_problem(B, H, W, oh, ow):
    rng = np.random.default_rng(B * 7919 + H * 1009 + W * 31 + oh + ow)
    cand = exact_pixels(H, W, oh, ow)
    s = np.empty((B, H * W, 21), f32)
    pow2 = upsample_kernel(H, W, oh, ow) == "resize_argmax_pow2_kernel"
    special = {19: last_slot_case(H, W, oh // H), 20: thread_order_case(H, W, oh // H)} if pow2 else {}
    for b in range(B):
        for c in range(21):
            k = b * 21 + c
            if special.get(k) is not None:
                s[b, :, c] = special[k].reshape(-1)
            else:
                s[b, :, c] = pattern_map(PATTERNS[k % len(PATTERNS)], H * W, 12, 1, rng, cand)
    return s.reshape(B, H, W, 21)


# ---------------------------------------------------------------------------------------------------------------- helpers
@pytest.fixture(scope="module")
def ctx():
    c = runtime.default_context()
    yield c
    torch.cuda.synchronize()
    c.check_errors()


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _ptr(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def assert_bits(got, want, what):
    """Bit-for-bit equality; NaNs compare by position only (the device writes the canonical NaN, numpy keeps the operand's)."""
    got, want = np.asarray(got, f32), np.asarray(want, f32)
    assert got.shape == want.shape, (got.shape, want.shape)
    gn, wn = np.isnan(got), np.isnan(want)
    bad = (gn != wn) | (~gn & (got.view(np.uint32) != want.view(np.uint32)))
    if bad.any():
        i = tuple(int(v[0]) for v in np.nonzero(bad))
        raise AssertionError("%s: %d of %d values differ, first at %s: got %r, want %r" % (what, int(bad.sum()), bad.size, i, got[i], want[i]))


def assert_same_bits(a, b, what):
    assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8)), what


def images_to_check(B):
    return sorted({0, B // 2, B - 1})


def run_resize(ctx, xg, oh, ow):
    B, H, W, Cc = xg.shape
    y = Guarded((B, oh, ow, Cc), torch.float32)
    _lib.check(ctx.lib.h3d_resize_bilinear_tf1(ctx.h, _ptr(xg), _ptr(y.t), B, H, W, Cc, oh, ow, _stream()), "h3d_resize_bilinear_tf1")
    return y.check("y")


def run_maxpool(ctx, xg):
    B, H, W, Cc = xg.shape
    y = Guarded((B, H // 2, W // 2, Cc), torch.float32)
    _lib.check(ctx.lib.h3d_maxpool2x2_f32(ctx.h, _ptr(xg), _ptr(y.t), B, H, W, Cc, _stream()), "h3d_maxpool2x2_f32")
    return y.check("y")


def run_avgpool(ctx, xg):
    B, H, W, Cc = xg.shape
    y = Guarded((B, H // 8, W // 8, Cc), torch.float32)
    _lib.check(ctx.lib.h3d_avgpool8(ctx.h, _ptr(xg), _ptr(y.t), B, H, W, Cc, _stream()), "h3d_avgpool8")
    return y.check("y")


def run_crop(ctx, img, center, scale, crop):
    B, H, W, Cc = img.shape
    y = Guarded((B, crop, crop, Cc), torch.float32)
    _lib.check(ctx.lib.h3d_crop_image_from_xy(ctx.h, _ptr(img), _ptr(center), _ptr(scale), _ptr(y.t), B, H, W, Cc, crop, _stream()),
               "h3d_crop_image_from_xy")
    return y.check("crop")


def run_detect(ctx, sg):
    B, H, W, Cc = sg.shape
    uv = Guarded((B, Cc, 2), torch.float32)         # int32 results in a float32 canary buffer: the canary is no valid index
    _lib.check(ctx.lib.h3d_detect_keypoints(ctx.h, _ptr(sg), B, H, W, Cc, _ptr(uv.t), _stream()), "h3d_detect_keypoints")
    return uv.check("uv").view(np.int32)


def run_upsample(ctx, sg, oh, ow, aligned=True):
    B, H, W, _ = sg.shape
    n = B * oh * ow * 21
    if aligned:
        up = Guarded((B, oh, ow, 21), torch.float32)
        t = up.t
    else:                       # one float past a 16-byte boundary
        up = Guarded((n + 1,), torch.float32)
        t = up.t[1:].view(B, oh, ow, 21)
        assert t.data_ptr() % 16 == 4
    uv = Guarded((B, 21, 2), torch.float32)
    _lib.check(ctx.lib.h3d_upsample_detect_keypoints(ctx.h, _ptr(sg), B, H, W, oh, ow, _ptr(t), _ptr(uv.t), _stream()),
               "h3d_upsample_detect_keypoints")
    if aligned:
        maps = up.check("scoremaps_up")
    else:                       # the float before the output keeps the canary
        maps = up.check("scoremaps_up", 1, n + 1)[1:].reshape(B, oh, ow, 21)
    return maps, uv.check("uv").view(np.int32)


# ---------------------------------------------------------------------------------------------------------------- resize
@pytest.mark.parametrize("case", RESIZE, ids=_id)
def test_resize(ctx, case):
    B, H, W, Cc, oh, ow, kernel = case
    assert resize_kernel(H, W, Cc, oh, ow) == kernel
    x = np.random.default_rng(B + H + W + Cc).normal(size=(B, H, W, Cc)).astype(f32)
    xg = _cu(x)
    y = run_resize(ctx, xg, oh, ow)
    assert_bits(y, T.resize_bilinear_tf1(x, oh, ow), "resize %s" % (case,))
    assert_same_bits(run_resize(ctx, xg, oh, ow), y, "a second run")
    for i in images_to_check(B):
        assert_same_bits(run_resize(ctx, _cu(x[i:i + 1]), oh, ow)[0], y[i], "image %d alone" % i)


# ---------------------------------------------------------------------------------------------------------------- pools
@pytest.mark.parametrize("case", MAXPOOL, ids=_id)
def test_maxpool(ctx, case):
    B, H, W, Cc, kernel = case
    assert maxpool_kernel(Cc) == kernel
    x = np.random.default_rng(H * W + Cc).normal(size=(B, H, W, Cc)).astype(f32)
    xg = _cu(x)
    y = run_maxpool(ctx, xg)
    assert_bits(y, T.max_pool_2x2(x), "max-pool %s" % (case,))
    assert_same_bits(run_maxpool(ctx, xg), y, "a second run")
    for i in images_to_check(B):
        assert_same_bits(run_maxpool(ctx, _cu(x[i:i + 1]))[0], y[i], "image %d alone" % i)


@pytest.mark.parametrize("case", AVGPOOL, ids=_id)
def test_avgpool8(ctx, case):
    B, H, W, Cc = case
    rng = np.random.default_rng(H + W + Cc)
    x = (rng.normal(size=(B, H, W, Cc)) * np.exp(rng.uniform(-4, 4, size=(B, H, W, Cc)))).astype(f32)   # a wide range of magnitudes
    win = x.astype(f64).reshape(B, H // 8, 8, W // 8, 8, Cc)
    mean, mag = win.mean(axis=(2, 4)), np.abs(win).sum(axis=(2, 4)) / 64
    xg = _cu(x)
    y = run_avgpool(ctx, xg)
    err = np.abs(y.astype(f64) - mean)
    assert (err <= GAMMA_63 * mag).all(), "worst |y - mean| / (gamma_63 mean|x|) = %.3f" % float((err / (GAMMA_63 * mag)).max())
    assert_same_bits(run_avgpool(ctx, xg), y, "a second run")
    for i in images_to_check(B):
        assert_same_bits(run_avgpool(ctx, _cu(x[i:i + 1]))[0], y[i], "image %d alone" % i)
    # integers in [-1000, 1000]: every partial sum is an integer below 2^24 and the division by 64 is exact
    xi = rng.integers(-1000, 1001, size=(B, H, W, Cc)).astype(f32)
    want = xi.astype(f64).reshape(B, H // 8, 8, W // 8, 8, Cc).mean(axis=(2, 4))
    assert np.array_equal(run_avgpool(ctx, _cu(xi)).astype(f64), want)


# ---------------------------------------------------------------------------------------------------------------- crop
def crop_samples(center, scale, n, crop):
    """The sample coordinates of one axis (n = H or W) of crop_and_resize after crop_image_from_xy's box arithmetic, in float32 as
    oracle.tf1_ops.crop_and_resize computes them"""
    ff = f32
    css = ff(crop) / ff(scale)
    half = np.floor(css / ff(2.0)).astype(ff)
    a = ff(center) - half
    an, bn = a / ff(n), (a + css) / ff(n)
    if crop == 1:
        return np.array([ff(0.5) * (an + bn) * ff(n - 1)], ff)
    step = (bn - an) * ff(n - 1) / ff(crop - 1)
    return (an * ff(n - 1) + np.arange(crop, dtype=ff) * step).astype(ff)


def edge_center(n, crop, scale, want):
    """A centre whose samples along an axis of n pixels hit `want`: "zero" / "top" (a sample exactly on 0 / n - 1), "below" / "above"
    (a sample in (-1/16, 0) / (n - 1, n - 1 + 1/16)), scanning centres in steps of 1/64."""
    for c in np.arange(-crop, n + crop, 1 / 64, dtype=f32):
        s = crop_samples(c, scale, n, crop)
        hit = {"zero": (s == 0).any(), "top": (s == f32(n - 1)).any(), "below": ((s < 0) & (s > -1 / 16)).any(),
               "above": ((s > f32(n - 1)) & (s < n - 1 + 1 / 16)).any()}[want]
        if hit:
            return float(c)
    raise AssertionError("no centre puts a sample %s for n=%d crop=%d scale=%g" % (want, n, crop, scale))


EDGE_TARGETS = [("zero", "top"), ("top", "zero"), ("below", "above"), ("above", "below")]    # (rows, columns) of images 0 .. 3


@functools.lru_cache(maxsize=None)
def crop_problem(B, H, W, Cc, crop, boxes):
    rng = np.random.default_rng(B + H * 7 + W * 11 + Cc * 13 + crop)
    img = rng.uniform(-0.5, 0.5, size=(B, H, W, Cc)).astype(f32)
    scale = np.array([CROP_SCALES[i % len(CROP_SCALES)] for i in range(B)], f32)
    if boxes == "random":
        center = np.stack([rng.uniform(-20, H + 20, B), rng.uniform(-20, W + 20, B)], 1).astype(f32)
    else:
        scale[:] = 1.0
        center = np.array([[edge_center(H, crop, 1.0, ty), edge_center(W, crop, 1.0, tx)] for ty, tx in EDGE_TARGETS[:B]], f32)
    return img, center, scale


@pytest.mark.parametrize("case", CROP, ids=_id)
def test_crop(ctx, case):
    B, H, W, Cc, crop, boxes, path = case
    assert crop_path(B, Cc, crop) == path
    img, center, scale = crop_problem(B, H, W, Cc, crop, boxes)
    ig, cg, sg = _cu(img), _cu(center), _cu(scale)
    y = run_crop(ctx, ig, cg, sg, crop)
    check = range(B) if B <= 16 else sorted({0, 1, B // 3, B // 2, B - 2, B - 1})
    for i in check:
        assert_bits(y[i], O.crop_image_from_xy(img[i:i + 1], center[i:i + 1], crop, scale[i:i + 1])[0], "crop of image %d" % i)
    assert_same_bits(run_crop(ctx, ig, cg, sg, crop), y, "a second run")
    for i in images_to_check(B):
        assert_same_bits(run_crop(ctx, _cu(img[i:i + 1]), _cu(center[i:i + 1]), _cu(scale[i:i + 1]), crop)[0], y[i], "image %d alone" % i)


# ---------------------------------------------------------------------------------------------------------------- arg-max
@pytest.mark.parametrize("case", DETECT, ids=_id)
def test_detect_keypoints(ctx, case):
    B, H, W, Cc = case
    P, gx = detect_grid(H, W, Cc)
    assert (H * W) % P or P == 1, "H W a multiple of P"
    s = detect_problem(B, H, W, Cc)
    sg = _cu(s)
    uv = run_detect(ctx, sg)
    want = argmax_uv(s)
    bad = np.nonzero((uv != want).any(-1))
    assert not bad[0].size, "%d maps differ, first (image %d, channel %d, pattern %s): got %s, want %s" % (
        bad[0].size, bad[0][0], bad[1][0], PATTERNS[(bad[0][0] * Cc + bad[1][0]) % len(PATTERNS)], uv[bad[0][0], bad[1][0]],
        want[bad[0][0], bad[1][0]])
    assert_same_bits(run_detect(ctx, sg), uv, "a second run")
    for i in images_to_check(B):
        assert_same_bits(run_detect(ctx, _cu(s[i:i + 1]))[0], uv[i], "image %d alone" % i)


@pytest.mark.parametrize("case", UPSAMPLE, ids=_id)
def test_upsample_detect_keypoints(ctx, case):
    B, H, W, oh, ow, aligned, kernel = case
    assert upsample_kernel(H, W, oh, ow, aligned) == kernel
    s = upsample_problem(B, H, W, oh, ow)
    sg = _cu(s)
    maps, uv = run_upsample(ctx, sg, oh, ow, aligned)
    ref = T.resize_bilinear_tf1(s, oh, ow)
    assert_bits(maps, ref, "up-sampled maps")
    want = argmax_uv(ref)
    bad = np.nonzero((uv != want).any(-1))
    assert not bad[0].size, "%d maps differ, first (image %d, channel %d): got %s, want %s" % (
        bad[0].size, bad[0][0], bad[1][0], uv[bad[0][0], bad[1][0]], want[bad[0][0], bad[1][0]])
    maps2, uv2 = run_upsample(ctx, sg, oh, ow, aligned)
    assert_same_bits(maps2, maps, "a second run (maps)")
    assert_same_bits(uv2, uv, "a second run (uv)")
    for i in images_to_check(B):
        mi, ui = run_upsample(ctx, _cu(s[i:i + 1]), oh, ow, aligned)
        assert_same_bits(mi[0], maps[i], "image %d alone (maps)" % i)
        assert_same_bits(ui[0], uv[i], "image %d alone (uv)" % i)


def test_find_max_location(ctx):
    """utils.general.find_max_location: the C = 1 arg-max of [B,H,W] maps, every pattern once"""
    from hand3d_b200.utils.general import find_max_location
    B, H, W = len(PATTERNS), 97, 203
    P, gx = detect_grid(H, W, 1)
    rng = np.random.default_rng(31)
    s = np.stack([pattern_map(k, H * W, P, gx, rng) for k in PATTERNS]).reshape(B, H, W)
    got = find_max_location(_cu(s)).cpu().numpy()
    np.testing.assert_array_equal(got, O.find_max_location(s))
    np.testing.assert_array_equal(got, argmax_uv(s[..., None])[:, 0])


def seg_logits(B, H, W, rng):
    """logits whose fg probability saturates to exactly 1.0 on plateaus: a band of rows across all the CTAs of an image (its first pixel
    late in the image) and a block before it at a lower value"""
    lg = np.zeros((B, H, W, 2), f32)
    lg[..., 0] = rng.normal(size=(B, H, W)).astype(f32)
    lg[..., 1] = lg[..., 0] - 2.0
    for b in range(B):
        r0 = H // 2 + b
        lg[b, r0:r0 + max(2, H // 8), W // 3:, 1] = 40.0        # fg = 1.0
        lg[b, 1:3, 1:4, 1] = lg[b, 1:3, 1:4, 0] + 3.0           # high fg, below 1.0
    return lg


@pytest.mark.parametrize("case", SEG, ids=_id)
def test_seg_max_loc_plateau(ctx, case):
    B, H, W = case
    lg = seg_logits(B, H, W, np.random.default_rng(H + W))
    fg, _ = O.seg_fg_det(lg)
    want = O.find_max_location(fg)
    assert (fg.reshape(B, -1).max(1) == 1.0).all() and all((fg[b] == 1.0).sum() > W for b in range(B))
    loc = Guarded((B, 2), torch.float32)
    center, scale = torch.empty((B, 2), device="cuda"), torch.empty((B, 1), device="cuda")
    lgg = _cu(lg)
    _lib.check(ctx.lib.h3d_seg_postprocess(ctx.h, _ptr(lgg), B, H, W, None, _ptr(loc.t), _ptr(center), None, _ptr(scale), _stream()),
               "h3d_seg_postprocess")
    got = loc.check("max_loc").view(np.int32)
    np.testing.assert_array_equal(got, want)
    from hand3d_b200.utils.general import find_max_location
    np.testing.assert_array_equal(find_max_location(_cu(fg)).cpu().numpy(), want)


# ---------------------------------------------------------------------------------------------------------------- 65 535 images
def test_max_grid_images_run(ctx):
    """MAX_GRID_IMAGES images in one call: the per-image grid rows of the crop and all arg-max kernels reach their limit"""
    B = MAX_GRID_IMAGES
    rng = np.random.default_rng(41)
    s = rng.normal(size=(B, 1, 3, 1)).astype(f32)
    np.testing.assert_array_equal(run_detect(ctx, _cu(s)), argmax_uv(s))
    img = rng.uniform(size=(B, 2, 2, 1)).astype(f32)
    center = rng.uniform(0, 2, size=(B, 2)).astype(f32)
    scale = np.ones(B, f32)
    y = run_crop(ctx, _cu(img), _cu(center), _cu(scale), 1)
    for i in (0, 1, B // 2, B - 1):
        assert_bits(y[i], O.crop_image_from_xy(img[i:i + 1], center[i:i + 1], 1, scale[i:i + 1])[0], "crop %d" % i)
    u = rng.normal(size=(B, 1, 1, 21)).astype(f32)
    maps, uv = run_upsample(ctx, _cu(u), 1, 2)
    assert_bits(maps, T.resize_bilinear_tf1(u, 1, 2), "up-sampled maps")
    assert (uv == 0).all()


# ---------------------------------------------------------------------------------------------------------------- refusals
def _refused(ctx, call, what, msg):
    """call() returns H3D_EINVAL with a message containing msg and enqueues no kernel"""
    n0 = ctx.launch_count
    rc = call()
    torch.cuda.synchronize()
    assert rc == _lib.EINVAL, "%s: rc %d" % (what, rc)
    assert msg in _lib.last_error(), (what, _lib.last_error())
    assert ctx.launch_count == n0, "%s enqueued a kernel" % what


BAD_RESIZE = [(0, 4, 4, 2, 8, 8), (1, 0, 4, 2, 8, 8), (1, 4, 0, 2, 8, 8), (1, 4, 4, 0, 8, 8), (1, 4, 4, 2, 0, 8), (1, 4, 4, 2, 8, 0),
              (1, -1, 4, 2, 8, 8), (1, 4, 4, 2, 8, -3)]
BAD_POOL = [(0, 8, 8, 4), (1, 1, 8, 4), (1, 8, 1, 4), (1, 8, 8, 0), (1, 0, 0, 4), (1, -8, 8, 4)]
BAD_AVGPOOL = [(0, 8, 8, 4), (1, 0, 8, 4), (1, 8, 0, 4), (1, 8, 8, 0), (1, -8, 8, 4)]
BAD_CROP = [(0, 4, 4, 3, 8), (1, 0, 4, 3, 8), (1, 4, 0, 3, 8), (1, 4, 4, 0, 8), (1, 4, 4, 3, 0), (1, 4, 4, 3, -1), (1, 4, 4, 3, 46341)]
BAD_DETECT = [(0, 4, 4, 21), (1, 0, 4, 21), (1, 4, 0, 21), (1, 4, 4, 0), (1, 4, 4, 257), (1, 65536, 65536, 1)]
BAD_UPSAMPLE = [(0, 4, 4, 32, 32), (1, 0, 4, 32, 32), (1, 4, 0, 32, 32), (1, 4, 4, 0, 32), (1, 4, 4, 32, 0), (1, 4, 4, 65536, 65536)]


def test_shapes_refused(ctx):
    buf = Guarded((4096,), torch.float32)
    p = _ptr(buf.t)
    L = ctx.lib
    for B, H, W, Cc, oh, ow in BAD_RESIZE:
        _refused(ctx, lambda: L.h3d_resize_bilinear_tf1(ctx.h, p, p, B, H, W, Cc, oh, ow, _stream()), "resize %s" % ((B, H, W, Cc, oh, ow),),
                 "h3d_resize_bilinear_tf1")
    for B, H, W, Cc in BAD_POOL:
        _refused(ctx, lambda: L.h3d_maxpool2x2_f32(ctx.h, p, p, B, H, W, Cc, _stream()), "max-pool %s" % ((B, H, W, Cc),), "h3d_maxpool2x2_f32")
    for B, H, W, Cc in BAD_AVGPOOL:
        _refused(ctx, lambda: L.h3d_avgpool8(ctx.h, p, p, B, H, W, Cc, _stream()), "avgpool8 %s" % ((B, H, W, Cc),), "h3d_avgpool8")
    for B, H, W, Cc, crop in BAD_CROP:
        _refused(ctx, lambda: L.h3d_crop_image_from_xy(ctx.h, p, p, p, p, B, H, W, Cc, crop, _stream()), "crop %s" % ((B, H, W, Cc, crop),),
                 "h3d_crop_image_from_xy")
    for B, H, W, Cc in BAD_DETECT:
        _refused(ctx, lambda: L.h3d_detect_keypoints(ctx.h, p, B, H, W, Cc, p, _stream()), "detect %s" % ((B, H, W, Cc),), "detect_keypoints")
    for B, H, W, oh, ow in BAD_UPSAMPLE:
        _refused(ctx, lambda: L.h3d_upsample_detect_keypoints(ctx.h, p, B, H, W, oh, ow, p, p, _stream()), "upsample %s" % ((B, H, W, oh, ow),),
                 "h3d_upsample_detect_keypoints")
    _refused(ctx, lambda: L.h3d_resize_bilinear_tf1(ctx.h, None, p, 1, 4, 4, 2, 8, 8, _stream()), "resize x NULL", "required")
    _refused(ctx, lambda: L.h3d_crop_image_from_xy(ctx.h, p, None, p, p, 1, 4, 4, 3, 8, _stream()), "crop center NULL", "required")
    _refused(ctx, lambda: L.h3d_detect_keypoints(ctx.h, p, 1, 4, 4, 21, None, _stream()), "detect uv NULL", "required")
    buf.check("the untouched buffer", 0, 0)


def test_batches_past_the_grid_refused(ctx):
    """MAX_GRID_IMAGES + 1 images: the crop, both arg-max entries and seg_postprocess refuse the call before anything is enqueued"""
    B = MAX_GRID_IMAGES + 1
    L = ctx.lib
    x = Guarded((B * 21 * 2,), torch.float32)
    out = Guarded((B * 21 * 2,), torch.float32)
    px, po = _ptr(x.t), _ptr(out.t)
    x.t.zero_()
    _refused(ctx, lambda: L.h3d_crop_image_from_xy(ctx.h, px, px, px, po, B, 1, 1, 1, 1, _stream()), "crop", "65535")
    _refused(ctx, lambda: L.h3d_detect_keypoints(ctx.h, px, B, 1, 1, 1, po, _stream()), "detect", "65535")
    _refused(ctx, lambda: L.h3d_upsample_detect_keypoints(ctx.h, px, B, 1, 1, 1, 1, po, po, _stream()), "upsample", "65535")
    _refused(ctx, lambda: L.h3d_seg_postprocess(ctx.h, px, B, 1, 1, None, None, po, None, po, _stream()), "seg_postprocess", "65535")
    out.check("the untouched output", 0, 0)


def test_runtime_wrappers_refuse_empty_tensors(ctx):
    """The runtime wrappers pass zero-size tensors (a NULL or a valid pointer) to the entries, which refuse them"""
    z = torch.zeros((1, 0, 4, 21), device="cuda")
    for fn in (lambda: ctx.resize_bilinear(z, 8, 8), lambda: ctx.max_pool(z), lambda: ctx.avg_pool8(z), lambda: ctx.detect_keypoints(z),
               lambda: ctx.upsample_detect_keypoints(z, 8, 8), lambda: ctx.crop_image_from_xy(z[..., :3], torch.zeros((1, 2), device="cuda"), 8,
                                                                                            torch.ones(1, device="cuda"))):
        with pytest.raises(RuntimeError, match="bad shape|required"):
            fn()


# ---------------------------------------------------------------------------------------------------------------- dispatch
NAME = {"copy": r"Memcpy DtoD"}


def dispatch_runs(ctx):
    """(callable, [kernel names in launch order]) for every row of every table whose kernel differs from the rows before it"""
    runs, seen = [], set()

    def once(key, fn, names):
        if key not in seen:
            seen.add(key)
            runs.append((fn, names))

    for B, H, W, Cc, oh, ow, kernel in RESIZE:
        xg = _cu(np.ones((B, H, W, Cc), f32))
        once(kernel, lambda a=(xg, oh, ow): run_resize(ctx, *a), [kernel])
    for B, H, W, Cc, kernel in MAXPOOL:
        xg = _cu(np.ones((B, H, W, Cc), f32))
        once(kernel, lambda a=xg: run_maxpool(ctx, a), [kernel])
    xg = _cu(np.ones(AVGPOOL[0], f32))
    once("avgpool8_kernel", lambda: run_avgpool(ctx, xg), ["avgpool8_kernel"])
    img, center, scale = crop_problem(*CROP[3][:6])
    cargs = (_cu(img), _cu(center), _cu(scale), CROP[3][4])
    once("crop_image_kernel", lambda: run_crop(ctx, *cargs), ["crop_image_kernel"])
    sg = _cu(detect_problem(*DETECT[3]))
    once("heatmap_argmax_kernel", lambda: run_detect(ctx, sg), ["heatmap_argmax_kernel", "argmax_decode_kernel"])
    for B, H, W, oh, ow, aligned, kernel in UPSAMPLE:
        ug = _cu(np.ones((B, H, W, 21), f32))
        once(kernel, lambda a=(ug, oh, ow, aligned): run_upsample(ctx, *a), [kernel, "argmax_decode_kernel"])
    B, H, W = SEG[0]
    lg = _cu(seg_logits(B, H, W, np.random.default_rng(0)))
    once("seg_prob_kernel<false>", lambda: ctx.seg_postprocess(lg), ["seg_prob_kernel<false>", "mask_grow_kernel"])
    return runs


def check_dispatch(ctx):
    from torch.profiler import ProfilerActivity, profile
    runs = dispatch_runs(ctx)
    for fn, _ in runs:                                         # warm-up outside the profiler
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for fn, _ in runs:
            fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memset" not in e.name
             and ("h3d::" in e.name or "Memcpy DtoD" in e.name)]
    want = [n for _, ns in runs for n in ns]
    ok = len(names) == len(want) and all(re.search(NAME.get(w, re.escape(w)), n) for w, n in zip(want, names))
    assert ok, "\n".join(["want %s" % want] + names)
    assert set(want) == set(expected_kernels()) | {"mask_grow_kernel"}
    return names


def test_dispatch():
    """check_dispatch in a child process, so that no profiler session runs in the suite's own process (see
    test_gpu_conv_direct_paths.test_dispatch)."""
    import subprocess
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "dispatch"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=600)
    assert r.returncode == 0 and "dispatch: " in r.stdout, "dispatch child failed:\n" + r.stdout[-6000:]


if __name__ == "__main__" and sys.argv[1:] == ["dispatch"]:
    _ctx = runtime.default_context()
    _names = check_dispatch(_ctx)
    torch.cuda.synchronize()
    _ctx.check_errors()
    print("dispatch: %d kernels" % len(_names))

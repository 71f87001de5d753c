"""The fp32 CUDA-core convolution (conv_direct_kernel, conv_splitk_reduce_kernel, conv3x3_c3_kernel) and fully connected layer
(fc_splitk_kernel + fc_reduce_kernel) on every path their launchers choose from the shape, the channel offsets and the alignment.

Each table entry is marked with the path it is meant to take: the kernel (c3_tc, c3_ffma, vec, scalar) and "+splitk" where K is split
over blockIdx.z and reduced by a second launch.  tests/test_conv_direct_coverage_cpu.py asks the library (h3d_conv2d_f32_geometry,
h3d_fully_connected_f32_geometry) which path each entry takes and fails when a path drops out; here every run also checks the launch
count, and test_dispatch the kernel names.  The operator entry h3d_conv2d_f32 reaches strides 1 to 3, split-K and the unaligned
input; route 1 of h3d_conv2d_layer_planes reaches Cin_total > Cin, channel offsets of the fp32 output and the plane epilogues.

Four kinds of check.  fp64 parity in the scale-relative metric of test_gpu_tc_range.py: |y - ref| / S, S = conv_SAME(|x|, |w|) + |b|.
Exact canaries: small-integer operands with a position code (every (image, row, column) has its own integers, every tap its own
weights), whose partial sums are integers below 2^24 and exact in any order, against the integer result; leaky ReLU restated in
float32.  Bit-for-bit identities: the vec and scalar gathers (same operands, same order), an image alone and in its batch, and each
plane against planes_oracle's encoding of the fp32 output.  Guards: every output and plane buffer is filled with a NaN canary and
followed by GUARD canary words, and every element outside the written channels must keep it."""
import ctypes as C
import functools
import os
import re
import sys

import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

HERE = os.path.dirname(os.path.abspath(__file__))
for _p in (os.path.dirname(HERE), HERE):        # the repository (also when run as the dispatch child) and tests/
    if _p not in sys.path:
        sys.path.insert(0, _p)
import planes_oracle as P  # noqa: E402
from hand3d_b200 import _lib, runtime  # noqa: E402
from oracle import tf1_ops as T  # noqa: E402

pytestmark = pytest.mark.gpu
f32, f64 = np.float32, np.float64

# max |y - ref| / S of the fp32 CUDA-core kernels, three times the largest an H100 (700 W) measured: 3.6e-7, entry 1x79x239x32 -> 64
# 3x3 (K = 288 in one pass, 2.4 million outputs); the layers 2.2e-7, the FC layers 1.7e-7 (DESIGN.md section 6.1)
BOUND = 1.1e-6
# the tensor-core first layer (c3_tc, planes only): test_gpu_tc_range.BOUND of its precision
TC_BOUND = {"bf16x3": 1e-5, "fp16x3": 3e-6}
CANARY32, CANARY16, CANARY8 = 0x7FC0A5A5, 0x7FA5, 0x7F    # NaN patterns no layer of finite operands writes (runtime.Context)
GUARD = 4096                                               # elements after each buffer that must keep the canary
ENTRY_SPLITK_PIXELS = 64 * 295                             # h3d_conv2d_f32 offers split-K scratch up to B Ho Wo = 64 x 295

# ---------------------------------------------------------------------------------------------------------------- shape tables
# h3d_conv2d_f32: (B, H, W, Cin, Cout, ksize, stride, x_aligned, path).  Cin_total = Cin, no offsets, fp32 output only.
ENTRY_SHAPES = [
    # kernel sizes 1, 3, 5, 7 at strides 1, 2, 3, even and odd H and W; Cout tails 1, 2, 3, 5, 21, 63, 65, 129
    (2, 9, 14, 16, 21, 1, 1, True, "vec"),
    (1, 10, 11, 16, 5, 1, 2, True, "vec"),
    (2, 11, 8, 32, 63, 3, 1, True, "vec+splitk"),
    (1, 12, 13, 21, 64, 3, 2, True, "scalar"),             # pad_t = 0, pad_l = 1
    (3, 13, 7, 3, 2, 3, 3, True, "scalar"),
    (1, 16, 15, 32, 65, 5, 2, True, "vec+splitk"),         # pad_t = 1, pad_l = 2
    (2, 14, 13, 16, 256, 5, 3, True, "vec+splitk"),
    (1, 8, 8, 21, 1, 5, 1, True, "scalar+splitk"),
    (2, 7, 9, 149, 129, 7, 1, True, "scalar+splitk"),      # K = 7301 in 58 slices
    (1, 9, 10, 149, 3, 7, 3, True, "scalar+splitk"),
    (2, 15, 16, 3, 64, 7, 2, True, "scalar"),
    (1, 6, 33, 16, 129, 3, 1, True, "vec"),
    # the first-layer kernel: ragged H and W, a last CTA of fewer than 4 tiles, tiles of one CTA in two images (B = 9)
    (2, 32, 32, 3, 64, 3, 1, True, "c3_ffma"),
    (2, 19, 45, 3, 64, 3, 1, True, "c3_ffma"),
    (1, 5, 7, 3, 64, 3, 1, True, "c3_ffma"),
    (9, 17, 40, 3, 64, 3, 1, True, "c3_ffma"),
    # one step outside it
    (2, 16, 16, 3, 64, 3, 2, True, "scalar"),
    (2, 9, 9, 3, 63, 3, 1, True, "scalar"),
    (1, 9, 9, 3, 65, 3, 1, True, "scalar"),
    # split-K on each side of its boundaries: Ktot 255 / 256; 295 / 296 CTAs with one and with several 64-channel tiles, the first
    # pair also B Ho Wo = 18880 / 18881 at the entry's scratch rule; a split count lowered by the rounding of k_per_split
    (2, 5, 7, 255, 21, 1, 1, True, "scalar"),
    (2, 5, 7, 256, 21, 1, 1, True, "vec+splitk"),
    (1, 118, 160, 32, 64, 3, 1, True, "vec+splitk"),
    (1, 79, 239, 32, 64, 3, 1, True, "vec"),
    (1, 59, 64, 16, 300, 5, 1, True, "vec+splitk"),
    (2, 64, 74, 32, 100, 3, 1, True, "vec"),
    (2, 40, 40, 160, 8, 3, 1, True, "vec+splitk"),         # 11 slices asked, k_per_split 144 -> 10
    # x one float past a 16-byte boundary: contiguous, not aligned -> the scalar gather
    (1, 9, 10, 16, 21, 3, 1, False, "scalar"),
    (2, 5, 7, 256, 21, 1, 1, False, "scalar+splitk"),
    (2, 11, 8, 32, 63, 3, 1, False, "scalar+splitk"),
]

# route 1 of h3d_conv2d_layer_planes (stride 1, cin_off 0, no split-K): (B, H, W, Cx, Cin, Cout, ksize, planes, Cy_total, cy_off,
# Cyf_total, cyf_off, path); planes None = fp32 output only, Cyf_total None = planes only.
LAYERS = [
    (2, 19, 45, 3, 3, 64, 3, "bf16x3", 72, 8, None, 0, "c3_tc"),
    (1, 9, 40, 3, 3, 64, 3, "fp16x3", 64, 0, None, 0, "c3_tc"),
    (2, 19, 45, 3, 3, 64, 3, "fp16x3", 64, 0, 72, 4, "c3_ffma"),        # fp32 output at cout_off % 4 == 0, Cout_total > 64
    (9, 17, 40, 3, 3, 64, 3, "fp16_f8c", 64, 0, None, 0, "c3_ffma"),
    (3, 9, 13, 3, 3, 64, 3, "bf16", 80, 16, 68, 4, "c3_ffma"),
    (1, 8, 33, 3, 3, 64, 3, None, 0, 0, 128, 64, "c3_ffma"),
    (2, 9, 13, 4, 3, 64, 3, None, 0, 0, 64, 0, "scalar"),                # Cin_total = 4
    (2, 9, 13, 3, 3, 64, 3, None, 0, 0, 70, 2, "scalar"),                # cout_off % 4 != 0
    (2, 9, 13, 3, 3, 64, 3, "bf16x3", 72, 4, None, 0, "scalar"),         # cs_off % 8 != 0
    # the plane epilogue of conv_direct_kernel at generic shapes, cs_off != 0
    (2, 9, 13, 32, 32, 21, 3, "bf16", 40, 3, 24, 1, "vec"),
    (1, 10, 11, 17, 16, 63, 5, "fp16", 70, 5, None, 0, "scalar"),        # Cx = Cin + 1
    (2, 7, 9, 152, 149, 65, 7, "fp16_f8c", 72, 7, 65, 0, "scalar"),
    (1, 12, 10, 48, 32, 129, 1, "bf16x3", 136, 2, 132, 3, "vec"),
    (2, 8, 9, 21, 21, 5, 3, "fp16x3", 8, 1, 5, 0, "scalar"),
    (1, 9, 9, 64, 16, 2, 1, "fp16_f8c", 3, 1, None, 0, "vec"),
    (2, 11, 7, 64, 64, 256, 5, "fp16x3", 264, 8, 256, 0, "vec"),
]

# h3d_fully_connected_f32: (B, in_features, out_features)
FC_SHAPES = [
    (1, 1, 1), (31, 30, 3), (32, 33, 63), (33, 512, 64), (64, 2050, 65), (65, 4098, 512), (160, 512, 512), (300, 2050, 63),
    (1, 4098, 512), (300, 33, 1), (160, 30, 65), (65, 1, 3), (31, 4098, 64), (33, 2050, 512), (1, 512, 3), (64, 4098, 1),
    (300, 4098, 512),
]


def _id(s):
    return "x".join(str(v) if isinstance(v, (int, np.integer)) else str(v) for v in s)


def entry_splitk_floats(B, H, W, stride):
    """The split-K scratch h3d_conv2d_f32 offers."""
    return _lib.CONV_SPLITK_SCRATCH_FLOATS if B * -(-H // stride) * -(-W // stride) <= ENTRY_SPLITK_PIXELS else 0


def entry_geometry(shape):
    B, H, W, Cin, Cout, k, s, aligned = shape[:8]
    return runtime.conv2d_f32_geometry(B, H, W, Cin, Cout, k, s, x_aligned=aligned,
                                       splitk_scratch_floats=entry_splitk_floats(B, H, W, s))


def layer_geometry(layer, yf=None):
    """yf overrides the layer's fp32 output (Cyf_total, cyf_off)."""
    B, H, W, Cx, Cin, Cout, k, planes, Cy_total, cy_off, Cyf_total, cyf_off = layer[:12]
    if yf is not None:
        Cyf_total, cyf_off = yf
    return runtime.conv2d_f32_geometry(B, H, W, Cin, Cout, k, 1, Cin_total=Cx, Cout_total=Cyf_total or Cout, cout_off=cyf_off,
                                       yf=Cyf_total is not None, planes=planes, Cs_total=Cy_total, cs_off=cy_off, splitk_scratch_floats=0)


def path_of(geometry):
    kernel, _, ksplit, _ = geometry
    return kernel + ("+splitk" if ksplit > 1 else "")


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


def _x_on_device(x, aligned=True):
    """x on the device, or at one float past a 16-byte boundary (a contiguous view into a larger buffer)."""
    if aligned:
        return _cu(x)
    flat = torch.empty(x.size + 4, dtype=torch.float32, device="cuda")
    view = flat[1:1 + x.size].view(x.shape)
    view.copy_(torch.from_numpy(np.ascontiguousarray(x)))
    assert view.data_ptr() % 16 == 4
    return view


class Guarded:
    """A device buffer of `shape` filled with the canary and followed by GUARD canary elements."""
    FILL = {torch.float32: (CANARY32, torch.int32), torch.int16: (CANARY16, torch.int16), torch.uint8: (CANARY8, torch.uint8)}

    def __init__(self, shape, dtype):
        self.n = int(np.prod(shape))
        self.flat = torch.empty(self.n + GUARD, dtype=dtype, device="cuda")
        fill, view = self.FILL[dtype]
        self.flat.view(view).fill_(fill)
        self.fill, self.bits = fill, view
        self.t = self.flat[:self.n].view(shape)

    def check(self, what, lo=None, hi=None):
        """Host copy of the buffer after asserting the guard and, for channel range [lo, hi), that exactly those channels were
        written (lo None: every element)."""
        raw = self.flat.view(self.bits).cpu().numpy()
        assert (raw[self.n:] == np.array(self.fill).astype(raw.dtype)).all(), "%s: %d elements written behind the buffer" % (
            what, int((raw[self.n:] != np.array(self.fill).astype(raw.dtype)).sum()))
        body = raw[:self.n].reshape(self.t.shape)
        canary = body == np.array(self.fill).astype(raw.dtype)
        if lo is None:
            assert not canary.any(), "%s: %d elements never written" % (what, int(canary.sum()))
        else:
            inside = np.zeros(body.shape[-1], bool)
            inside[lo:hi] = True
            assert not canary[..., inside].any(), "%s: %d elements of channels [%d, %d) never written" % (
                what, int(canary[..., inside].sum()), lo, hi)
            assert canary[..., ~inside].all(), "%s: %d elements outside channels [%d, %d) overwritten" % (
                what, int((~canary[..., ~inside]).sum()), lo, hi)
        return self.t.cpu().numpy()


def scale_rel_err(y, ref, S):
    return float((np.abs(np.asarray(y, f64) - ref) / S).max())


def leaky_f32(v):
    """fmaxf(v, 0.01f v) in float32, as the epilogues compute it."""
    v = np.asarray(v, f32)
    return np.maximum(v, f32(0.01) * v)


@functools.lru_cache(maxsize=None)
def float_problem(B, H, W, Cx, Cin, Cout, k, stride):
    """x ~ N(0, 1) over Cx channels (the layer reads the first Cin), w ~ N(0, 1 / K), b ~ N(0, 1); the fp64 result and its bound S."""
    rng = np.random.default_rng(81)
    x = rng.normal(size=(B, H, W, Cx)).astype(f32)
    w = (rng.normal(size=(k, k, Cin, Cout)) / np.sqrt(k * k * Cin)).astype(f32)
    b = rng.normal(size=Cout).astype(f32)
    xs = x[..., :Cin].astype(f64)
    ref = T.conv2d_same(xs, w.astype(f64), b.astype(f64), stride, f64)
    S = T.conv2d_same(np.abs(xs), np.abs(w.astype(f64)), np.abs(b.astype(f64)), stride, f64)
    return x, w, b, ref, S


@functools.lru_cache(maxsize=None)
def int_problem(B, H, W, Cx, Cin, Cout, k, stride):
    """Position code x[b,h,w,c] = ((1 + pixel index) (c + 1) mod 251) - 125 and random weights in [-2, 2], biases in [-8, 8]:
    |partial sums| <= 125 x 2 x 7301 + 8 < 2^24.  Returns the exact result as float64 (integers below 2^53)."""
    rng = np.random.default_rng(82)
    idx = (1 + np.arange(B * H * W, dtype=np.int64)).reshape(B, H, W, 1)
    x = ((idx * (1 + np.arange(Cx, dtype=np.int64))) % 251 - 125).astype(f32)
    w = rng.integers(-2, 3, size=(k, k, Cin, Cout)).astype(f32)
    b = rng.integers(-8, 9, size=Cout).astype(f32)
    assert 125 * 2 * k * k * Cin + 8 < 2 ** 24
    ref = T.conv2d_same(x[..., :Cin].astype(f64), w.astype(f64), b.astype(f64), stride, f64)
    return x, w, b, ref


def assert_exact(got, want, what):
    want = np.asarray(want, f64)
    assert got.shape == want.shape
    bad = np.asarray(got, f64) != want
    if bad.any():
        i = tuple(int(v[0]) for v in np.nonzero(bad))
        raise AssertionError("%s: %d of %d values differ, first at %s: got %r, want %r" % (what, int(bad.sum()), bad.size, i, got[i], want[i]))


def run_entry(ctx, xg, w, b, Cout, k, stride, leaky, geometry):
    """h3d_conv2d_f32 into a guarded buffer; checks the launch count against the query's split."""
    B, H, W, Cin = xg.shape
    Ho, Wo = -(-H // stride), -(-W // stride)
    y = Guarded((B, Ho, Wo, Cout), torch.float32)
    n0 = ctx.launch_count
    _lib.check(ctx.lib.h3d_conv2d_f32(ctx.h, _ptr(xg), _ptr(w), _ptr(b), _ptr(y.t), B, H, W, Cin, Cout, k, stride, int(leaky),
                                      _stream()), "h3d_conv2d_f32")
    assert ctx.launch_count - n0 == (2 if geometry[2] > 1 else 1), "launches of %s" % (geometry,)
    return y.check("y")


def run_layer(ctx, x, w, b, layer, leaky, yf=None):
    """route 1 of h3d_conv2d_layer_planes with guarded buffers: (planes dict (all four, to see which were written), fp32 output).
    yf overrides the layer's fp32 output (Cyf_total, cyf_off)."""
    B, H, W, Cx, Cin, Cout, k, planes, Cy_total, cy_off, Cyf_total, cyf_off = layer[:12]
    if yf is not None:
        Cyf_total, cyf_off = yf
    out = {}
    if planes:
        out.update(hi=Guarded((B, H, W, Cy_total), torch.int16), lo=Guarded((B, H, W, Cy_total), torch.int16),
                   l8=Guarded((B, H, W, Cy_total), torch.uint8), h8=Guarded((B, H, W, Cy_total), torch.uint8))
    if Cyf_total:
        out["yf"] = Guarded((B, H, W, Cyf_total), torch.float32)
    n0 = ctx.launch_count
    ctx.conv_layer(_cu(x), w, b, planes or "bf16x3", route=1, leaky=leaky, planes=bool(planes), Cy_total=Cy_total, cy_off=cy_off,
                   yf=bool(Cyf_total), Cyf_total=Cyf_total, cyf_off=cyf_off, out={key: g.t for key, g in out.items()})
    geometry = layer_geometry(layer, yf)
    assert ctx.launch_count - n0 == (2 if geometry[2] > 1 else 1)
    got = {}
    for key in ("hi", "lo", "l8", "h8"):
        if key in out:
            if key in P.PLANES[planes]:
                got[key] = out[key].check(key, cy_off, cy_off + Cout).view(np.uint8 if key in ("l8", "h8") else np.uint16)
            else:
                out[key].check(key, 0, 0)          # a plane the precision does not use is never written
    yf_host = out["yf"].check("yf", cyf_off, cyf_off + Cout) if "yf" in out else None
    return got, yf_host


def planes_of(got, planes, cy_off, Cout):
    return {key: v[..., cy_off:cy_off + Cout] for key, v in got.items() if key in P.PLANES[planes]}


def assert_planes_encode(got, yf, planes, what):
    """Each plane is planes_oracle's encoding of the fp32 output, bit for bit."""
    want = P.encode(np.asarray(yf, f32), planes)
    for key in P.PLANES[planes]:
        bad = got[key] != want[key]
        assert not bad.any(), "%s: %s plane differs from the encoding of yf at %d of %d values, first at %s" % (
            what, key, int(bad.sum()), bad.size, tuple(int(v[0]) for v in np.nonzero(bad)))


# ---------------------------------------------------------------------------------------------------------------- operator entry
@pytest.mark.parametrize("shape", ENTRY_SHAPES, ids=_id)
def test_entry_vs_fp64(ctx, shape):
    B, H, W, Cin, Cout, k, s, aligned, path = shape
    geometry = entry_geometry(shape)
    assert path_of(geometry) == path, "%s runs %s" % (shape, geometry)
    x, w, b, ref, S = float_problem(B, H, W, Cin, Cin, Cout, k, s)
    xg, wg, bg = _x_on_device(x, aligned), _cu(w), _cu(b)
    for leaky in (False, True):
        y = run_entry(ctx, xg, wg, bg, Cout, k, s, leaky, geometry)
        e = scale_rel_err(y, T.leaky_relu(ref) if leaky else ref, S)
        print("F32ERR entry/%s/%s %.3e" % (_id(shape), "leaky" if leaky else "linear", e))
        assert e < BOUND, "scale-relative error %.3e, bound %.1e" % (e, BOUND)


@pytest.mark.parametrize("shape", ENTRY_SHAPES, ids=_id)
def test_entry_exact_canary(ctx, shape):
    B, H, W, Cin, Cout, k, s, aligned, _ = shape
    x, w, b, ref = int_problem(B, H, W, Cin, Cin, Cout, k, s)
    xg, wg, bg = _x_on_device(x, aligned), _cu(w), _cu(b)
    geometry = entry_geometry(shape)
    assert_exact(run_entry(ctx, xg, wg, bg, Cout, k, s, False, geometry), ref, "y[b,h,w,co]")
    assert_exact(run_entry(ctx, xg, wg, bg, Cout, k, s, True, geometry), leaky_f32(ref), "leaky y[b,h,w,co]")


@pytest.mark.parametrize("shape", [s for s in ENTRY_SHAPES if s[3] % 16 == 0 and s[7]], ids=_id)
def test_vec_and_scalar_gathers_agree(ctx, shape):
    """The same layer from an aligned and an unaligned x: the float4 and the scalar gather read the same operands into the same K
    order, so the outputs agree bit for bit, with split-K and without."""
    B, H, W, Cin, Cout, k, s, _, _ = shape
    g_vec, g_scalar = entry_geometry(shape), entry_geometry(shape[:7] + (False,))
    assert g_vec[0] == "vec" and g_scalar[0] == "scalar" and g_vec[1:] == g_scalar[1:]
    x, w, b, _, _ = float_problem(B, H, W, Cin, Cin, Cout, k, s)
    wg, bg = _cu(w), _cu(b)
    y_vec = run_entry(ctx, _x_on_device(x, True), wg, bg, Cout, k, s, True, g_vec)
    y_scalar = run_entry(ctx, _x_on_device(x, False), wg, bg, Cout, k, s, True, g_scalar)
    assert np.array_equal(y_vec.view(np.uint32), y_scalar.view(np.uint32))


def _batch_independent(shape):
    return shape[0] > 1 and entry_geometry((1,) + shape[1:])[2:] == entry_geometry(shape)[2:]


@pytest.mark.parametrize("shape", [s for s in ENTRY_SHAPES if _batch_independent(s)], ids=_id)
def test_entry_image_does_not_depend_on_the_batch(ctx, shape):
    """With the same split of K, image i run alone equals image i of the batch, bit for bit: the first, the last, and for the first
    layer an image whose tiles share a CTA with the image before it."""
    B, H, W, Cin, Cout, k, s, aligned, _ = shape
    x, w, b, _, _ = float_problem(B, H, W, Cin, Cin, Cout, k, s)
    wg, bg = _cu(w), _cu(b)
    y = run_entry(ctx, _x_on_device(x, aligned), wg, bg, Cout, k, s, True, entry_geometry(shape))
    for i in sorted({0, B // 2, B - 1}):
        y1 = run_entry(ctx, _x_on_device(x[i:i + 1], aligned), wg, bg, Cout, k, s, True, entry_geometry((1,) + shape[1:]))
        assert np.array_equal(y1[0].view(np.uint32), y[i].view(np.uint32)), "image %d of %d" % (i, B)


# ---------------------------------------------------------------------------------------------------------------- layer (route 1)
def _check_yf_kernel(layer, yf):
    """The fp32 output added for the bit-identity checks keeps the layer on its kernel."""
    assert layer_geometry(layer, yf)[0] == layer_geometry(layer)[0] or layer[-1] == "c3_tc"


def _identity_yf(layer):
    """An fp32 output to add to a planes-only layer that keeps it on its kernel: c3_ffma at an aligned offset, the generic kernels at
    an odd one.  (c3_tc has no fp32 output: adding one moves it to c3_ffma.)"""
    Cout = layer[5]
    return (Cout + 4, 4) if layer[-1] == "c3_ffma" else (Cout + 1, 1)


@pytest.mark.parametrize("layer", LAYERS, ids=_id)
def test_layer_vs_fp64(ctx, layer):
    B, H, W, Cx, Cin, Cout, k, planes, Cy_total, cy_off, Cyf_total, cyf_off, path = layer
    assert path_of(layer_geometry(layer)) == path
    x, w, b, ref, S = float_problem(B, H, W, Cx, Cin, Cout, k, 1)
    ref = T.leaky_relu(ref)
    got, yf = run_layer(ctx, x, w, b, layer, True)
    if yf is not None:
        e = scale_rel_err(yf[..., cyf_off:cyf_off + Cout], ref, S)
        print("F32ERR layer/%s %.3e" % (_id(layer), e))
        assert e < BOUND, "scale-relative error %.3e, bound %.1e" % (e, BOUND)
    if not planes:
        return
    pl = planes_of(got, planes, cy_off, Cout)
    if path == "c3_tc":
        d = P.decode(pl, planes)
        bound = TC_BOUND[planes] * S + P.FORMAT_REL[planes] * np.abs(ref) + P.FORMAT_ABS[planes]
        assert (np.abs(d - ref) <= bound).all(), "decoded planes: worst excess %.3e" % float((np.abs(d - ref) - bound).max())
        return
    if yf is None:          # planes only: the same kernel with an fp32 output too writes the same planes
        yfo = _identity_yf(layer)
        _check_yf_kernel(layer, yfo)
        got2, yf = run_layer(ctx, x, w, b, layer, True, yf=yfo)
        cyf_off = yfo[1]
        for key in pl:
            assert np.array_equal(planes_of(got2, planes, cy_off, Cout)[key], pl[key]), "%s plane changed with an fp32 output" % key
    assert_planes_encode(pl, yf[..., cyf_off:cyf_off + Cout], planes, "layer %s" % _id(layer))


@pytest.mark.parametrize("layer", LAYERS, ids=_id)
def test_layer_exact_canary(ctx, layer):
    """Integer operands: the fp32 output is the exact result (leaky restated in float32) and every plane its encoding; planes-only
    layers are checked through their planes alone."""
    B, H, W, Cx, Cin, Cout, k, planes, Cy_total, cy_off, Cyf_total, cyf_off, path = layer
    x, w, b, ref = int_problem(B, H, W, Cx, Cin, Cout, k, 1)
    for leaky in (False, True):
        want = leaky_f32(ref) if leaky else ref.astype(f32)
        got, yf = run_layer(ctx, x, w, b, layer, leaky)
        if yf is not None:
            assert_exact(yf[..., cyf_off:cyf_off + Cout], want, "yf[b,h,w,co], leaky %s" % leaky)
        if planes:
            assert_planes_encode(planes_of(got, planes, cy_off, Cout), want, planes, "integer layer %s, leaky %s" % (_id(layer), leaky))


# ---------------------------------------------------------------------------------------------------------------- fully connected
def run_fc(ctx, x, w, b, leaky):
    B, n_in = x.shape
    n_out = w.shape[1]
    xg, wg, bg = _cu(x), _cu(w), _cu(b)          # held until the call returns: a freed tensor's memory would be reused
    y = Guarded((B, n_out), torch.float32)
    n0 = ctx.launch_count
    _lib.check(ctx.lib.h3d_fully_connected_f32(ctx.h, _ptr(xg), _ptr(wg), _ptr(bg), _ptr(y.t), B, n_in, n_out, int(leaky), _stream()),
               "h3d_fully_connected_f32")
    assert ctx.launch_count - n0 == 2
    return y.check("y")


@pytest.mark.parametrize("shape", FC_SHAPES, ids=_id)
def test_fc_vs_fp64(ctx, shape):
    B, n_in, n_out = shape
    rng = np.random.default_rng(83)
    x = rng.normal(size=(B, n_in)).astype(f32)
    w = (rng.normal(size=(n_in, n_out)) / np.sqrt(n_in)).astype(f32)
    b = rng.normal(size=n_out).astype(f32)
    ref = x.astype(f64) @ w.astype(f64) + b
    S = np.abs(x.astype(f64)) @ np.abs(w.astype(f64)) + np.abs(b.astype(f64))
    for leaky in (False, True):
        e = scale_rel_err(run_fc(ctx, x, w, b, leaky), T.leaky_relu(ref) if leaky else ref, S)
        print("F32ERR fc/%s/%s %.3e" % (_id(shape), "leaky" if leaky else "linear", e))
        assert e < BOUND, "scale-relative error %.3e, bound %.1e" % (e, BOUND)


@pytest.mark.parametrize("shape", FC_SHAPES, ids=_id)
def test_fc_exact_canary(ctx, shape):
    """x[b, i] = ((b + 1) (i + 1) mod 251) - 125, weights in [-2, 2]: every row and every K slice has its own integers."""
    B, n_in, n_out = shape
    rng = np.random.default_rng(84)
    x = (((1 + np.arange(B, dtype=np.int64))[:, None] * (1 + np.arange(n_in, dtype=np.int64))) % 251 - 125).astype(f32)
    w = rng.integers(-2, 3, size=(n_in, n_out)).astype(f32)
    b = rng.integers(-8, 9, size=n_out).astype(f32)
    ref = x.astype(f64) @ w.astype(f64) + b
    assert_exact(run_fc(ctx, x, w, b, False), ref, "y[b,o]")
    assert_exact(run_fc(ctx, x, w, b, True), leaky_f32(ref), "leaky y[b,o]")


# ---------------------------------------------------------------------------------------------------------------- dispatch
DISPATCH = {"vec": r"conv_direct_kernel<true", "scalar": r"conv_direct_kernel<false", "c3_ffma": r"conv3x3_c3_kernel",
            "c3_tc": r"conv_c3_tc_kernel"}


def check_dispatch(ctx):
    """One entry and one layer per path, then a fully connected layer, under one profiler session: the kernel names, in launch
    order, are the paths the query reports, with conv_splitk_reduce_kernel after the partial sums exactly when K is split."""
    runs, want = [], []
    for s in (ENTRY_SHAPES[0], ENTRY_SHAPES[2], ENTRY_SHAPES[3], ENTRY_SHAPES[7], ENTRY_SHAPES[14], ENTRY_SHAPES[-3]):
        B, H, W, Cin, Cout, k, st, aligned, path = s
        x, w, b, _, _ = float_problem(B, H, W, Cin, Cin, Cout, k, st)
        args = (_x_on_device(x, aligned), _cu(w), _cu(b), Cout, k, st, True, entry_geometry(s))
        runs.append(lambda a=args: run_entry(ctx, *a))
        want.append(path)
    for layer in (LAYERS[0], LAYERS[3], LAYERS[8]):
        B, H, W, Cx, Cin, Cout, k = layer[:7]
        x, w, b, _, _ = float_problem(B, H, W, Cx, Cin, Cout, k, 1)
        runs.append(lambda a=(x, w, b, layer): run_layer(ctx, *a, True))
        want.append(layer[-1])
    assert set(want) == {"vec", "vec+splitk", "scalar", "scalar+splitk", "c3_ffma", "c3_tc"}
    xf = np.ones((33, 512), f32)
    runs.append(lambda: run_fc(ctx, xf, np.ones((512, 64), f32), np.zeros(64, f32), False))
    for fn in runs:                                            # warm-up outside the profiler
        fn()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for fn in runs:
            fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and ("conv" in e.name or "fc_" in e.name)]
    patterns = [p for path in want for p in [DISPATCH[path.split("+")[0]]] + (["conv_splitk_reduce_kernel"] if "+" in path else [])]
    patterns += ["fc_splitk_kernel", "fc_reduce_kernel"]
    assert len(names) == len(patterns) and all(re.search(p, n) for p, n in zip(patterns, names)), "\n".join(
        ["want %s" % patterns] + names)
    return names


def test_dispatch():
    """check_dispatch in a child process, so that no profiler session runs in the suite's own process: there, a session of this
    module was followed, several modules later, by test_gpu_native_size.py::test_dispatch seeing none of its kernels under the
    profiler.  The other profiler tests of the suite each expect a process whose first profiler session is their own."""
    import subprocess
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "dispatch"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=600)
    assert r.returncode == 0 and "dispatch: 13 kernels" in r.stdout, "dispatch child failed:\n" + r.stdout[-6000:]


if __name__ == "__main__" and sys.argv[1:] == ["dispatch"]:
    _ctx = runtime.default_context()
    _names = check_dispatch(_ctx)
    torch.cuda.synchronize()
    _ctx.check_errors()
    print("dispatch: %d kernels" % len(_names))

"""The training kernels of csrc/train.cu and csrc/train_lift.cu on every path their launchers take.

Each table row is marked with the path the launcher picks from the shape alone, restated in tests/train_order_oracle.py
(resize_grad_passes, scoremap_chunks, xent_blocks, mse_blocks, grid_for, adam_chunk_prefix); test_dispatch runs one row per kernel
under torch.profiler and checks the names, and tests/test_train_paths_coverage_cpu.py checks without a GPU that every __global__ of
the two files is reached by some row or excluded with a reason, and that the tables reach every case below.

Every sum in these kernels runs in an order fixed by the shape, in __fadd_rn / __fmul_rn / __fdiv_rn / __fsqrt_rn, so the resize
gradient, the score-map loss, the MSE (each with its gradient) and Adam are compared bit for bit with their float32 restatements
(tests/train_order_oracle.py, train_oracle.adam_tf_f32), and with the fp64 oracles within bounds.  The cross-entropy evaluates expf
and logf, which numpy cannot restate, so it is held to a bound from fp64 and to an exact canary.  Exact canaries on integer-valued
inputs make every dropped or repeated term visible: a pixel, a chunk, a block or a finalising lap.

Every run writes into buffers filled with a NaN canary and followed by guard words (test_gpu_conv_direct_paths.Guarded), and every
row runs twice and must give the same bits."""
import ctypes as C
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
import lift_train_oracle as L  # noqa: E402
import train_oracle as O  # noqa: E402
import train_order_oracle as R  # noqa: E402
from test_gpu_conv_direct_paths import CANARY32, GUARD, Guarded  # noqa: E402
import test_gpu_postprocess_paths as Pp  # noqa: E402
from test_gpu_postprocess_paths import _cu, _ptr, _stream, images_to_check  # noqa: E402

pytestmark = pytest.mark.gpu
f32, f64 = np.float32, np.float64
gamma = R.gamma
# Cross-entropy against fp64 (expf / logf are not restated): 3x the largest errors measured over XENT x XENT_LABELS on an H100
# 80GB HBM3 at 700 W (DESIGN 4.8): the loss 3.6e-8 scale-relative (xent_scale), the gradient 1.7e-7 normwise
XENT_TOL_LOSS = 3 * 3.7e-8
XENT_TOL_GRAD = 3 * 1.7e-7


def assert_bits(got, want, what):
    """test_gpu_postprocess_paths.assert_bits, also for the 0-d losses"""
    Pp.assert_bits(np.atleast_1d(got), np.atleast_1d(want), what)


def assert_same_bits(a, b, what):
    Pp.assert_same_bits(np.atleast_1d(a), np.atleast_1d(b), what)


# ---------------------------------------------------------------------------------------------------------------- paths
KERNEL = {"copy": "copy", "rows": "resize_grad_rows_kernel", "cols<21>": "resize_grad_cols_kernel<21>",
          "cols<2>": "resize_grad_cols_kernel<2>", "cols<0>": "resize_grad_cols_kernel<0>"}


def resize_grad_path(H, W, C_, oh, ow):
    """launch_resize_bilinear_tf1_grad: the copy, or the column pass (its template instance) and / or the row pass"""
    passes = R.resize_grad_passes(H, W, oh, ow)
    if not passes:
        return "copy"
    inst = C_ if C_ in (21, 2) else 0
    return "+".join("cols<%d>" % inst if p == "cols" else "rows" for p, _ in passes)


def resize_grad_loops(B, H, W, C_, oh, ow):
    """The passes of a row whose outputs outnumber one grid (grid_for caps it at 132 x 32 blocks of 256): the grid-stride loop"""
    return {p for p, n in R.resize_grad_passes(H, W, oh, ow) if B * n * C_ > R.grid_for(B * n * C_, 256) * 256}


def scoremap_path(B, H, W):
    """launch_scoremap_loss: the chunks per image (and why one), a short last chunk, idle pixel groups, finalize laps over B 21"""
    HW = H * W
    n = R.scoremap_chunks(B, HW)
    ppc = R.cdiv(HW, n)
    tags = ["1 chunk (HW <= 256)" if HW <= 256 else "1 chunk (B >= 264)"] if n == 1 else ["%d chunks" % n]
    if n > 1 and HW - (n - 1) * ppc < ppc:
        tags.append("short last")
    if HW - (n - 1) * ppc < R.SM_GROUPS:
        tags.append("idle groups")
    if B * 21 > R.RED_THREADS:
        tags.append("laps")
    return ", ".join(tags)


def reduction_path(n):
    """xent_blocks / mse_blocks: blocks x items per block, and finalize laps over more than 256 partials"""
    nblk, per = R.reduction_blocks(n)
    return "%d x %d%s" % (nblk, per, ", laps" if nblk > R.RED_THREADS else "")


# ---------------------------------------------------------------------------------------------------------------- tables
# h3d_resize_bilinear_tf1_backward: (B, H, W, C, out_h, out_w, path); (H, W) the forward's input, (out_h, out_w) its output
RESIZE_GRAD = [
    (3, 32, 32, 21, 256, 256, "cols<21>+rows"),       # x8 up, PoseNet's
    (2, 30, 30, 21, 97, 97, "cols<21>+rows"),         # non-integer up
    (2, 17, 23, 21, 5, 7, "cols<21>+rows"),           # non-integer down
    (2, 16, 12, 21, 16, 29, "cols<21>"),              # only W changes
    (2, 16, 12, 21, 7, 12, "rows"),                   # only H changes
    (1, 1, 1, 21, 5, 5, "cols<21>+rows"),             # one input pixel
    (1, 256, 256, 21, 32, 32, "cols<21>+rows"),       # x1/8: the row pass has 1.4M outputs, the grid-stride loop
    (2, 8, 8, 21, 8, 8, "copy"),
    (2, 40, 40, 2, 320, 320, "cols<2>+rows"),         # x8 up, HandSegNet's
    (2, 64, 48, 2, 17, 13, "cols<2>+rows"),           # non-integer down
    (2, 16, 40, 2, 16, 13, "cols<2>"),                # only W changes, down
    (2, 9, 7, 2, 36, 7, "rows"),                      # only H changes, up
    (2, 9, 11, 2, 1, 1, "cols<2>+rows"),              # one output pixel
    (1, 3, 1000, 2, 3, 3, "cols<2>"),                 # 1000 -> 3 in W
    (2, 5, 3, 2, 5, 3, "copy"),
    (2, 12, 10, 3, 30, 17, "cols<0>+rows"),           # non-integer up
    (2, 48, 64, 1, 24, 32, "cols<0>+rows"),           # exact x1/2
    (1, 1, 1, 3, 7, 9, "cols<0>+rows"),               # one input pixel
    (2, 9, 11, 64, 1, 1, "cols<0>+rows"),             # one output pixel
    (2, 16, 12, 1, 16, 29, "cols<0>"),                # only W changes, up
    (1, 3, 3, 1, 3, 1000, "cols<0>"),                 # 3 -> 1000 in W
    (1, 1000, 2, 3, 3, 2, "rows"),                    # 1000 -> 3 in H
    (2, 1, 9, 64, 4, 9, "rows"),                      # one input row
    (1, 48, 48, 64, 384, 384, "cols<0>+rows"),        # the column pass has 1.2M outputs: the grid-stride loop
    (3, 5, 7, 1, 5, 7, "copy"),
    (1, 9, 9, 64, 9, 9, "copy"),
]

# h3d_scoremap_loss_forward / _backward: (B, H, W, path)
SCOREMAP = [
    (1, 1, 1, "1 chunk (HW <= 256), idle groups"),
    (1, 2, 3, "1 chunk (HW <= 256), idle groups"),
    (1, 10, 10, "1 chunk (HW <= 256)"),
    (8, 16, 16, "1 chunk (HW <= 256)"),
    (13, 10, 10, "1 chunk (HW <= 256), laps"),
    (13, 1, 257, "2 chunks, short last, laps"),
    (1, 256, 256, "256 chunks"),
    (8, 256, 256, "33 chunks, short last"),
    (265, 17, 17, "1 chunk (B >= 264), laps"),
    (65536, 1, 1, "1 chunk (HW <= 256), idle groups, laps"),     # more images than a grid has rows
    (70001, 2, 3, "1 chunk (HW <= 256), idle groups, laps"),
]
SCOREMAP_KINDS = ["binary", "fractional", "canary"]

# h3d_softmax_xent_forward / _backward: (rows, path)
XENT = [(1, "1 x 1"), (255, "1 x 255"), (2048, "1 x 2048"), (2049, "2 x 1025"), (524288, "256 x 2048"),
        (2097152, "1024 x 2048, laps"), (2097153, "1024 x 2049, laps"), (3000001, "1024 x 2930, laps")]
XENT_LABELS = ["one_hot", "soft", "unnormalised"]

# h3d_mse_loss_forward / _backward: (n, path)
MSE = [(1, "1 x 1"), (255, "1 x 255"), (504, "1 x 504"), (2048, "1 x 2048"), (2049, "2 x 1025"), (2 ** 21, "1024 x 2048, laps"),
       (2 ** 21 + 1, "1024 x 2049, laps"), (3000007, "1024 x 2930, laps")]

# h3d_adam_step: (name, [(numel, (param, grad, m, v) float offsets from a 16-byte boundary)])
_MIS = [(8193 + 5 * i, tuple(off if a == i // 3 else 0 for a in range(4))) for i, off in enumerate([1, 2, 3] * 4)]
ADAM = [
    ("several chunks per block", [(4500000, (0, 0, 0, 0)), (300003, (0, 0, 0, 0)), (77, (0, 0, 0, 0))]),
    ("chunk edges", [(n, (0, 0, 0, 0)) for n in (0, 1, 3, 4, 8191, 8192, 8193, 16387, 0)]),
    ("1024 tensors", [((i * 37) % 301 + (8193 if i % 100 == 7 else 0), (0, 0, 0, 0)) for i in range(1024)]),
    ("one misaligned array", [(8192, (0, 0, 0, 0))] + _MIS[:6] + [(5000, (0, 0, 0, 0))] + _MIS[6:] + [(4, (0, 0, 0, 0))]),
    ("one element", [(1, (0, 0, 0, 0))]),
]
# optim.Adam over parameter views at float offsets: (numel, offset)
ADAM_OPTIM = [(8193, 1), (3, 2), (16387, 3), (1, 0), (8192, 0), (5, 1)]

# h3d_bone_rel_trafo_inv_backward (one thread per (sample, chain), blocks of 128) and h3d_rotate_canonical_backward
BONE_B = [1, 21, 22, 43, 1000]
ROTATE_B = [6, 70001]


def _id(s):
    return "x".join(str(v) for v in s) if isinstance(s, tuple) else str(s)


def expected_kernels():
    """{kernel name: rows} over every table"""
    out = {}
    for r in RESIZE_GRAD:
        for p in r[-1].split("+"):
            out.setdefault(KERNEL[p], []).append(r)
    for r in SCOREMAP:
        for k in ("scoremap_sq_partial_kernel", "scoremap_loss_finalize_kernel", "scoremap_loss_grad_kernel"):
            out.setdefault(k, []).append(r)
    for r in XENT:
        for k in ("xent_partial_kernel", "xent_finalize_kernel", "xent_grad_kernel"):
            out.setdefault(k, []).append(r)
    for r in MSE:
        for k in ("mse_partial_kernel", "mse_finalize_kernel", "mse_grad_kernel"):
            out.setdefault(k, []).append(r)
    for r in ADAM:
        out.setdefault("adam_step_kernel", []).append(r[0])
    for b in BONE_B:
        out.setdefault("bone_rel_trafo_inv_backward_kernel", []).append(b)
    for b in ROTATE_B:
        out.setdefault("rotate_canonical_backward_kernel", []).append(b)
    return out


# ---------------------------------------------------------------------------------------------------------------- helpers
@pytest.fixture(scope="module")
def ctx():
    c = runtime.default_context()
    yield c
    torch.cuda.synchronize()
    c.check_errors()


def _scalar(g):
    return None if g is None else torch.tensor(g, dtype=torch.float32, device="cuda")


def _err(g, ref):
    ref = np.asarray(ref, f64)
    return float(np.abs(np.asarray(g, f64) - ref).max() / max(np.abs(ref).max(), 1e-30))


def run_resize_grad(ctx, dyg, H, W):
    B, oh, ow, Cc = dyg.shape
    dx = Guarded((B, H, W, Cc), torch.float32)
    _lib.check(ctx.lib.h3d_resize_bilinear_tf1_backward(ctx.h, _ptr(dyg), _ptr(dx.t), B, H, W, Cc, oh, ow, _stream()),
               "h3d_resize_bilinear_tf1_backward")
    return dx.check("dx")


def run_scoremap(ctx, Pg, Tg, visg):
    B, H, W, _ = Pg.shape
    loss, rms = Guarded((), torch.float32), Guarded((B, 21), torch.float32)
    _lib.check(ctx.lib.h3d_scoremap_loss_forward(ctx.h, _ptr(Pg), _ptr(Tg), _ptr(visg), B, H, W, _ptr(loss.t), _ptr(rms.t), _stream()),
               "h3d_scoremap_loss_forward")
    return loss.check("loss")[()], rms.check("rms")


def run_scoremap_grad(ctx, Pg, Tg, visg, rmsg, g):
    B, H, W, _ = Pg.shape
    dP = Guarded(tuple(Pg.shape), torch.float32)
    _lib.check(ctx.lib.h3d_scoremap_loss_backward(ctx.h, _ptr(Pg), _ptr(Tg), _ptr(visg), _ptr(rmsg), _ptr(_scalar(g)), B, H, W, _ptr(dP.t),
                                                  _stream()), "h3d_scoremap_loss_backward")
    return dP.check("dpred")


def run_xent(ctx, xg, lg):
    loss = Guarded((), torch.float32)
    _lib.check(ctx.lib.h3d_softmax_xent_forward(ctx.h, _ptr(xg), _ptr(lg), xg.shape[0], _ptr(loss.t), _stream()), "h3d_softmax_xent_forward")
    return loss.check("loss")[()]


def run_xent_grad(ctx, xg, lg, g):
    d = Guarded(tuple(xg.shape), torch.float32)
    _lib.check(ctx.lib.h3d_softmax_xent_backward(ctx.h, _ptr(xg), _ptr(lg), _ptr(_scalar(g)), xg.shape[0], _ptr(d.t), _stream()),
               "h3d_softmax_xent_backward")
    return d.check("dlogits")


def run_mse(ctx, pg, qg):
    loss = Guarded((), torch.float32)
    _lib.check(ctx.lib.h3d_mse_loss_forward(ctx.h, _ptr(pg), _ptr(qg), pg.numel(), _ptr(loss.t), _stream()), "h3d_mse_loss_forward")
    return loss.check("loss")[()]


def run_mse_grad(ctx, pg, qg, g):
    d = Guarded(tuple(pg.shape), torch.float32)
    _lib.check(ctx.lib.h3d_mse_loss_backward(ctx.h, _ptr(pg), _ptr(qg), _ptr(_scalar(g)), pg.numel(), _ptr(d.t), _stream()),
               "h3d_mse_loss_backward")
    return d.check("dpred")


# ---------------------------------------------------------------------------------------------------------------- resize gradient
@pytest.mark.parametrize("case", RESIZE_GRAD, ids=_id)
def test_resize_backward(ctx, case):
    B, H, W, Cc, oh, ow, path = case
    assert resize_grad_path(H, W, Cc, oh, ow) == path
    dy = np.random.default_rng(B + H * 7 + W * 11 + Cc * 13 + oh).normal(size=(B, oh, ow, Cc)).astype(f32)
    dyg = _cu(dy)
    dx = run_resize_grad(ctx, dyg, H, W)
    assert_bits(dx, R.resize_grad(dy, H, W), "resize gradient %s" % (case,))
    e = _err(dx, O.resize_bilinear_grad(dy, H, W))
    assert e <= 1e-6, e
    assert_same_bits(run_resize_grad(ctx, dyg, H, W), dx, "a second run")
    for i in images_to_check(B):
        assert_same_bits(run_resize_grad(ctx, _cu(dy[i:i + 1]), H, W)[0], dx[i], "image %d alone" % i)


# ---------------------------------------------------------------------------------------------------------------- score-map loss
def scoremap_problem(B, H, W, kind):
    rng = np.random.default_rng(B * 31 + H * W + len(kind))
    if kind == "canary":
        # P - T = +-c[b,k] over each map, small integers with H W c^2 < 2^24; rms = |c| exactly
        cmax = min(5, int(np.sqrt((2 ** 24 - 1) / (H * W))))
        c = rng.integers(-cmax, cmax + 1, size=(B, 21)).astype(f32)
        T = rng.integers(-4, 5, size=(B, H, W, 21)).astype(f32)
        sign = np.where(rng.uniform(size=(B, H, W, 21)) < 0.5, 1, -1).astype(f32)
        P = T + sign * c[:, None, None, :]
        vis = (rng.uniform(size=(B, 21)) < 0.7).astype(f32)
        return P, T, vis, c
    P = rng.normal(size=(B, H, W, 21)).astype(f32)
    T = rng.normal(size=(B, H, W, 21)).astype(f32)
    T[0, :, :, 3] = P[0, :, :, 3]                              # rms == 0 for one map
    vis = (rng.uniform(size=(B, 21)) < 0.7).astype(f32)
    if kind == "fractional":
        vis = (vis * rng.uniform(0.05, 1.5, size=(B, 21))).astype(f32)
    return P, T, vis, None


@pytest.mark.parametrize("kind", SCOREMAP_KINDS)
@pytest.mark.parametrize("case", SCOREMAP, ids=_id)
def test_scoremap_loss(ctx, case, kind):
    B, H, W, path = case
    assert scoremap_path(B, H, W) == path
    P, T, vis, c = scoremap_problem(B, H, W, kind)
    Pg, Tg, vg = _cu(P), _cu(T), _cu(vis)
    loss, rms = run_scoremap(ctx, Pg, Tg, vg)
    want_loss, want_rms = R.scoremap_loss(P, T, vis)
    assert_bits(rms, want_rms, "rms")
    assert_bits(loss, want_loss, "loss")
    l2, r2 = run_scoremap(ctx, Pg, Tg, vg)
    assert_same_bits(l2, loss, "a second run (loss)")
    assert_same_bits(r2, rms, "a second run (rms)")
    ref_loss, ref_rms = O.scoremap_loss(P, T, vis)
    e_rms, e_loss, e_grad = R.scoremap_bounds(B, H * W)
    assert (np.abs(rms - ref_rms) <= e_rms * ref_rms).all()
    assert abs(float(loss) - ref_loss) <= e_loss * abs(ref_loss)
    if kind == "canary":
        assert np.array_equal(rms, np.abs(c))
        num = (vis * np.abs(c)).astype(f64).sum()
        assert num < 2 ** 24 and loss == f32(f32(num) / f32(f32(vis.astype(f64).sum()) + f32(0.001)))
    else:
        assert rms[0, 3] == 0
    rg = _cu(rms)
    for g in (None, -3.5):
        dP = run_scoremap_grad(ctx, Pg, Tg, vg, rg, g)
        assert_bits(dP, R.scoremap_loss_grad(P, T, vis, rms, g), "dpred, g %s" % g)
        assert_same_bits(run_scoremap_grad(ctx, Pg, Tg, vg, rg, g), dP, "a second run (dpred, g %s)" % g)
        ref = O.scoremap_loss_grad(P, T, vis, 1.0 if g is None else g)
        assert np.abs(dP - ref).max() <= e_grad * np.abs(ref).max()
        if kind != "canary":
            assert not dP[0, :, :, 3].any()                    # rms == 0
        assert not dP.transpose(0, 3, 1, 2)[vis == 0].any()


# ---------------------------------------------------------------------------------------------------------------- cross-entropy
def xent_problem(rows, labels):
    rng = np.random.default_rng(rows + len(labels))
    x = (rng.normal(size=(rows, 2)) * 4).astype(f32)
    big = rng.uniform(size=rows) < 0.1
    x[big] = rng.uniform(-80, 80, size=(int(big.sum()), 2)).astype(f32)          # logits up to +-80
    eq = rng.uniform(size=rows) < 0.05
    x[eq, 1] = x[eq, 0]                                                           # equal logits
    if labels == "one_hot":
        h = rng.uniform(size=rows) < 0.3
        lab = np.stack([~h, h], 1).astype(f32)
    else:
        lab = rng.uniform(size=(rows, 2)).astype(f32)
        if labels == "soft":
            lab = (lab / lab.sum(1, keepdims=True)).astype(f32)
    return x, lab


def xent_scale(x, lab):
    """The scale a row's loss is computed at: its labels times (1 + |x0 - x1|) (log s is in [0, log 2], -(x - m) in [0, |x0 - x1|]);
    the mean over the rows.  A row whose loss is a rounding of log s near 1 has a large relative error but a small one at this scale."""
    x, lab = x.astype(f64), lab.astype(f64)
    return float(((np.abs(lab[:, 0]) + np.abs(lab[:, 1])) * (1 + np.abs(x[:, 0] - x[:, 1]))).mean())


@pytest.mark.parametrize("labels", XENT_LABELS)
@pytest.mark.parametrize("case", XENT, ids=_id)
def test_softmax_xent(ctx, case, labels):
    rows, path = case
    assert reduction_path(rows) == path
    x, lab = xent_problem(rows, labels)
    xg, lg = _cu(x), _cu(lab)
    loss = run_xent(ctx, xg, lg)
    assert_same_bits(run_xent(ctx, xg, lg), loss, "a second run")
    e_loss = abs(float(loss) - O.softmax_xent(x, lab)) / xent_scale(x, lab)
    e_grad = 0.0
    for g in (None, 0.25):
        d = run_xent_grad(ctx, xg, lg, g)
        assert_same_bits(run_xent_grad(ctx, xg, lg, g), d, "a second run (dlogits, g %s)" % g)
        e_grad = max(e_grad, _err(d, O.softmax_xent_grad(x, lab, 1.0 if g is None else g)))
    print("cross-entropy %d rows, %s: loss %.2e scale-relative, gradient %.2e normwise" % (rows, labels, e_loss, e_grad))
    assert e_loss <= XENT_TOL_LOSS and e_grad <= XENT_TOL_GRAD, (e_loss, e_grad)


def test_xent_canary_arithmetic(ctx):
    """The exact canary's premise on the device: logits (0, -200) give expf(0) = 1, expf(-200) = 0 and logf(1) = 0, so a row with
    labels (0, 1) loses exactly 200 and its gradient is exactly (1, -1)"""
    xg, lg = _cu(np.array([[0.0, -200.0]], f32)), _cu(np.array([[0.0, 1.0]], f32))
    assert run_xent(ctx, xg, lg) == 200.0
    assert np.array_equal(run_xent_grad(ctx, xg, lg, None), np.array([[1.0, -1.0]], f32))


@pytest.mark.parametrize("case", XENT, ids=_id)
def test_softmax_xent_exact_canary(ctx, case):
    """Every row (0, -200): a row loses exactly 200 label_1.  label_1 small integers, mostly 0, 200 sum label_1 < 2^24: the total is
    an exact integer and the loss that integer over f32(rows), rounded once.  A dropped or repeated row, block or lap changes it."""
    rows, _ = case
    rng = np.random.default_rng(rows)
    x = np.tile(np.array([0.0, -200.0], f32), (rows, 1))
    lab = np.zeros((rows, 2), f32)
    lab[:, 0] = rng.integers(0, 2, rows)
    hit = rng.uniform(size=rows) < min(1.0, 20000 / rows)
    hit[-1] = True                                                                # the last row counts
    lab[hit, 1] = rng.integers(1, 3, int(hit.sum()))
    total = 200 * lab[:, 1].astype(f64).sum()
    assert total < 2 ** 24
    xg, lg = _cu(x), _cu(lab)
    assert run_xent(ctx, xg, lg) == f32(f32(total) / f32(rows))
    scale = f32(f32(-1.5) / f32(rows))
    d = run_xent_grad(ctx, xg, lg, -1.5)
    assert_bits(d, np.stack([scale * (f32(1) - lab[:, 0]), scale * (f32(0) - lab[:, 1])], 1), "dlogits")


# ---------------------------------------------------------------------------------------------------------------- MSE
@pytest.mark.parametrize("case", MSE, ids=_id)
def test_mse(ctx, case):
    n, path = case
    assert reduction_path(n) == path
    rng = np.random.default_rng(n)
    p, q = rng.normal(size=(2, n)).astype(f32)
    pg, qg = _cu(p), _cu(q)
    loss = run_mse(ctx, pg, qg)
    assert_bits(loss, R.mse(p, q), "loss")
    assert_same_bits(run_mse(ctx, pg, qg), loss, "a second run")
    assert abs(float(loss) - L.mse(p, q)) <= gamma(R.cdiv(R.reduction_blocks(n)[1], 256) + 8 + 4 + 8 + 3) * L.mse(p, q)
    for g in (None, -2.5):
        d = run_mse_grad(ctx, pg, qg, g)
        assert_bits(d, R.mse_grad(p, q, g), "dpred, g %s" % g)
        assert_same_bits(run_mse_grad(ctx, pg, qg, g), d, "a second run (dpred)")
    # integers: p - q small, sum (p - q)^2 < 2^24, so every partial sum is exact
    pi = rng.integers(-5, 6, n).astype(f32)
    qi = pi + rng.integers(-2, 3, n).astype(f32)
    want = ((pi.astype(f64) - qi) ** 2).sum()
    assert want < 2 ** 24
    assert run_mse(ctx, _cu(pi), _cu(qi)) == f32(f32(want) / f32(n))


# ---------------------------------------------------------------------------------------------------------------- Adam
PRE = 16          # canary floats before each Adam array (64 bytes: the arrays' 16-byte boundary, then the offset)


class AdamTensor:
    """param, grad, m, v of one table entry, each at its own float offset from a 16-byte boundary, between canary words"""

    def __init__(self, n, offsets, rng):
        self.n, self.offsets, self.bufs, self.views = n, offsets, [], []
        init = [rng.normal(size=n), rng.normal(size=n), rng.normal(size=n) * 0.1, rng.uniform(size=n) * 0.01]
        for off, a in zip(offsets, init):
            flat = torch.empty(PRE + n + GUARD, dtype=torch.float32, device="cuda")
            flat.view(torch.int32).fill_(CANARY32)
            v = flat[PRE + off:PRE + off + n]
            v.copy_(torch.from_numpy(a.astype(f32)))
            assert v.data_ptr() % 16 == 4 * off
            self.bufs.append((flat, PRE + off))
            self.views.append(v)

    def row(self):
        return [v.data_ptr() for v in self.views] + [self.n]

    def host(self):
        return [v.cpu().numpy() for v in self.views]          # param, grad, m, v

    def check_guards(self, what):
        for (flat, lo), name in zip(self.bufs, ("param", "grad", "m", "v")):
            raw = flat.view(torch.int32).cpu().numpy()
            outside = np.concatenate([raw[:lo], raw[lo + self.n:]])
            assert (outside == CANARY32).all(), "%s: %s written outside its %d elements" % (what, name, self.n)


def _adam_steps(ctx, tensors, steps, rng):
    """Steps the tensors through ctx.adam_step with hand-built tables and checks every element, the beta powers and the ticket after
    every call against train_oracle.adam_tf_f32; the learning rate changes before the second step"""
    table = torch.tensor([t.row() for t in tensors], dtype=torch.int64).cuda()
    state = torch.zeros(_lib.ADAM_STATE_WORDS, dtype=torch.float32, device="cuda")
    lr = 1e-3
    ctx.adam_state_set(state, lr, 0.9, 0.999)
    ref = [t.host() for t in tensors]
    for s in range(steps):
        if s == 1:
            lr = 3e-4
            ctx.adam_set_lr(state, lr)
        for t, r in zip(tensors, ref):
            gnew = (rng.normal(size=t.n) * (1e-6 if s == 2 else 1.0)).astype(f32)
            t.views[1].copy_(torch.from_numpy(gnew))
            r[1] = gnew
        ctx.adam_step(table, len(tensors), state, 0.9, 0.999, 1e-8)
        b1p, b2p = O.beta_powers_after(s)
        for i, (t, r) in enumerate(zip(tensors, ref)):
            r[0], r[2], r[3] = O.adam_tf_f32(r[0], r[1], r[2], r[3], lr, b1p, b2p)
            got = t.host()
            for k, name in ((0, "param"), (2, "m"), (3, "v")):
                assert_bits(got[k], r[k], "step %d, tensor %d (%d elements, offsets %s): %s" % (s, i, t.n, t.offsets, name))
        st = state.cpu()
        want = O.beta_powers_after(s + 1)
        assert st[0].item() == f32(lr) and (st[1].item(), st[2].item()) == (float(want[0]), float(want[1])), (s, st)
        assert st.view(torch.int32)[3].item() == 0, "the ticket after step %d" % s
    for i, t in enumerate(tensors):
        t.check_guards("tensor %d" % i)


@pytest.mark.parametrize("name,sizes", ADAM, ids=[a[0].replace(" ", "_") for a in ADAM])
def test_adam_step(ctx, name, sizes):
    rng = np.random.default_rng(len(sizes))
    tensors = [AdamTensor(n, off, rng) for n, off in sizes]
    _adam_steps(ctx, tensors, 3, rng)


def test_adam_optim_on_parameter_views(ctx):
    """optim.Adam takes any contiguous fp32 parameter: views at float offsets 1 to 3 run the scalar path, beside aligned ones"""
    from hand3d_b200.optim import Adam
    rng = np.random.default_rng(51)
    bases = [torch.zeros(n + 4, device="cuda") for n, _ in ADAM_OPTIM]
    params = []
    for base, (n, off) in zip(bases, ADAM_OPTIM):
        p = torch.nn.Parameter(base[off:off + n])
        p.data.copy_(torch.from_numpy(rng.normal(size=n).astype(f32)))
        assert p.data_ptr() % 16 == 4 * off and p.is_contiguous()
        params.append(p)
    opt = Adam(params, lr=1e-3)
    ref = [(p.detach().cpu().numpy(), np.zeros(p.numel(), f32), np.zeros(p.numel(), f32)) for p in params]
    lr = 1e-3
    for s in range(4):
        if s == 2:
            lr = 5e-4
            opt.set_lr(lr)
        grads = [rng.normal(size=p.numel()).astype(f32) for p in params]
        for p, g in zip(params, grads):
            p.grad = _cu(g)
        opt.step()
        b1p, b2p = O.beta_powers_after(s)
        ref = [O.adam_tf_f32(rp, g, rm, rv, lr, b1p, b2p) for (rp, rm, rv), g in zip(ref, grads)]
        for p, (rp, rm, rv) in zip(params, ref):
            assert_bits(p.detach().cpu().numpy(), rp, "param of %d at offset %d" % (p.numel(), (p.data_ptr() % 16) // 4))
            assert_bits(opt.state[p]["m"].cpu().numpy(), rm, "m")
            assert_bits(opt.state[p]["v"].cpu().numpy(), rv, "v")
        assert opt.beta_powers() == tuple(float(v) for v in O.beta_powers_after(s + 1))
        assert opt._dev_state.view(torch.int32)[3].item() == 0
    for base, (n, off) in zip(bases, ADAM_OPTIM):
        outside = torch.cat([base[:off], base[off + n:]])
        assert not outside.any(), "written outside the parameter view"


def test_adam_table_sizes_refused(ctx):
    """0 and 1025 tensors: H3D_EINVAL before anything is enqueued; the state is untouched"""
    t = AdamTensor(4, (0, 0, 0, 0), np.random.default_rng(0))
    table = torch.tensor([t.row()] * 1025, dtype=torch.int64).cuda()
    state = torch.zeros(_lib.ADAM_STATE_WORDS, dtype=torch.float32, device="cuda")
    ctx.adam_state_set(state, 1e-3, 0.9, 0.999)
    before = [a.copy() for a in t.host()]
    for n in (0, 1025):
        torch.cuda.synchronize()
        n0 = ctx.launch_count
        rc = ctx.lib.h3d_adam_step(ctx.h, _ptr(table), n, _ptr(state), C.c_float(0.9), C.c_float(0.999), C.c_float(1e-8), _stream())
        torch.cuda.synchronize()
        assert rc == _lib.EINVAL, (n, rc)
        assert "1 to 1024 tensors" in _lib.last_error()
        assert ctx.launch_count == n0
    for a, b in zip(t.host(), before):
        assert_same_bits(a, b, "a tensor of a refused call")
    assert state.cpu().tolist()[:3] == [f32(1e-3), f32(0.9), f32(0.999)]


# ---------------------------------------------------------------------------------------------------------------- adjoints
def run_bone_backward(ctx, relg, dg):
    B = relg.shape[0]
    d_rel = Guarded((B, 21, 3), torch.float32)
    _lib.check(ctx.lib.h3d_bone_rel_trafo_inv_backward(ctx.h, _ptr(relg), _ptr(dg), _ptr(d_rel.t), B, _stream()),
               "h3d_bone_rel_trafo_inv_backward")
    return d_rel.check("d_rel")


@pytest.mark.parametrize("B", BONE_B)
def test_bone_rel_trafo_inv_backward(ctx, B):
    """One thread per (sample, chain) in blocks of 128: B = 21 fills one block but two threads, 22 and 43 spill into the next"""
    rng = np.random.default_rng(B)
    rel = np.concatenate([rng.uniform(0.1, 1.0, (B, 21, 1)), rng.uniform(-1.5, 1.5, (B, 21, 2))], 2).astype(f32)
    d = rng.normal(size=(B, 21, 3)).astype(f32)
    relg, dg = _cu(rel), _cu(d)
    got = run_bone_backward(ctx, relg, dg)
    assert _err(got, L.bone_rel_trafo_inv_grad(rel, d)) <= 1e-5
    assert_same_bits(run_bone_backward(ctx, relg, dg), got, "a second run")
    for i in images_to_check(B):
        assert_same_bits(run_bone_backward(ctx, _cu(rel[i:i + 1]), _cu(d[i:i + 1]))[0], got[i], "sample %d alone" % i)


def run_rotate_backward(ctx, cg, ug, hg, og, rg):
    B = cg.shape[0]
    d_can, d_u = Guarded((B, 21, 3), torch.float32), Guarded((B, 3), torch.float32)
    _lib.check(ctx.lib.h3d_rotate_canonical_backward(ctx.h, _ptr(cg), _ptr(ug), _ptr(hg), _ptr(og), _ptr(rg), B, _ptr(d_can.t), _ptr(d_u.t),
                                                     _stream()), "h3d_rotate_canonical_backward")
    return d_can.check("d_can"), d_u.check("d_uxyz")


TIES = np.array([[1, 0], [0, 1], [0.5, 0.5], [0, 0], [1, 1], [-2, -2]], f32)      # rows 2 .. 5 tie: a left hand, as the forward


@pytest.mark.parametrize("B", ROTATE_B)
def test_rotate_canonical_backward(ctx, B):
    rng = np.random.default_rng(B)
    can = rng.normal(size=(B, 21, 3)).astype(f32)
    u = rng.normal(size=(B, 3)).astype(f32)
    hs = TIES[np.arange(B) % len(TIES)]
    d_out, d_R = rng.normal(size=(B, 21, 3)).astype(f32), rng.normal(size=(B, 3, 3)).astype(f32)
    args = [_cu(a) for a in (can, u, hs, d_out, d_R)]
    d_can, d_u = run_rotate_backward(ctx, *args)
    ref_c, ref_u = L.rotate_canonical_grad(can, u, hs, d_out, d_R)
    assert _err(d_can, ref_c) <= 1e-6 and _err(d_u, ref_u) <= 1e-4, (_err(d_can, ref_c), _err(d_u, ref_u))
    c2, u2 = run_rotate_backward(ctx, *args)
    assert_same_bits(c2, d_can, "a second run (d_can)")
    assert_same_bits(u2, d_u, "a second run (d_uxyz)")
    # a tie is a left hand: the same bits as hand_side (1, 0)
    left = hs.copy()
    left[(hs[:, 0] == hs[:, 1])] = (1, 0)
    cl, ul = run_rotate_backward(ctx, args[0], args[1], _cu(left), args[3], args[4])
    assert_same_bits(cl, d_can, "ties as left hands (d_can)")
    assert_same_bits(ul, d_u, "ties as left hands (d_uxyz)")
    for i in images_to_check(B):
        ci, ui = run_rotate_backward(ctx, *[a[i:i + 1] for a in args])
        assert_same_bits(ci[0], d_can[i], "sample %d alone" % i)
        assert_same_bits(ui[0], d_u[i], "sample %d alone" % i)


# ---------------------------------------------------------------------------------------------------------------- dispatch
NAME = {"copy": r"Memcpy DtoD"}


def dispatch_runs(ctx):
    """(callable, [kernel names in launch order]) for one row of each distinct path"""
    runs, seen = [], set()
    for B, H, W, Cc, oh, ow, path in RESIZE_GRAD:
        if path not in seen and B * H * W * Cc < 10 ** 6:
            seen.add(path)
            dyg = _cu(np.ones((B, oh, ow, Cc), f32))
            runs.append((lambda a=(dyg, H, W): run_resize_grad(ctx, *a), [KERNEL[p] for p in path.split("+")]))
    P, T, vis, _ = scoremap_problem(2, 8, 8, "binary")
    Pg, Tg, vg = _cu(P), _cu(T), _cu(vis)
    rg = _cu(R.scoremap_loss(P, T, vis)[1])
    runs.append((lambda: run_scoremap(ctx, Pg, Tg, vg), ["scoremap_sq_partial_kernel", "scoremap_loss_finalize_kernel"]))
    runs.append((lambda: run_scoremap_grad(ctx, Pg, Tg, vg, rg, None), ["scoremap_loss_grad_kernel"]))
    xg, lg = (_cu(a) for a in xent_problem(3000, "soft"))
    runs.append((lambda: run_xent(ctx, xg, lg), ["xent_partial_kernel", "xent_finalize_kernel"]))
    runs.append((lambda: run_xent_grad(ctx, xg, lg, None), ["xent_grad_kernel"]))
    pg, qg = _cu(np.ones(3000, f32)), _cu(np.zeros(3000, f32))
    runs.append((lambda: run_mse(ctx, pg, qg), ["mse_partial_kernel", "mse_finalize_kernel"]))
    runs.append((lambda: run_mse_grad(ctx, pg, qg, None), ["mse_grad_kernel"]))
    t = AdamTensor(100, (0, 0, 0, 0), np.random.default_rng(0))
    table = torch.tensor([t.row()], dtype=torch.int64).cuda()
    state = torch.zeros(_lib.ADAM_STATE_WORDS, dtype=torch.float32, device="cuda")
    ctx.adam_state_set(state, 1e-3, 0.9, 0.999)
    runs.append((lambda: ctx.adam_step(table, 1, state, 0.9, 0.999, 1e-8), ["adam_step_kernel"]))
    rel = _cu(np.full((3, 21, 3), 0.5, f32))
    runs.append((lambda: run_bone_backward(ctx, rel, rel), ["bone_rel_trafo_inv_backward_kernel"]))
    can, u, hs = _cu(np.ones((2, 21, 3), f32)), _cu(np.ones((2, 3), f32)), _cu(TIES[:2])
    runs.append((lambda: run_rotate_backward(ctx, can, u, hs, can, None), ["rotate_canonical_backward_kernel"]))
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
    assert set(want) == set(expected_kernels())
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

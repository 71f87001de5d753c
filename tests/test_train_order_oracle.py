"""The float32 order restatements of tests/train_order_oracle.py against the fp64 oracles (tests/train_oracle.py,
tests/lift_train_oracle.py), without a GPU: on random inputs within the error bound of each order, on integer-valued inputs exactly.
This keeps the restatement an independent check of each loss, not a copy of its kernel.

Bounds: a float32 sum through k roundings of terms x_i is within gamma_k sum |x_i| of the exact sum (train_order_oracle.gamma); k is
the longest chain of roundings a term passes through in the kernel's order, plus the rounding of the operations around the sum."""
import numpy as np
import pytest

import lift_train_oracle as L
import train_oracle as O
import train_order_oracle as R

f32, f64 = np.float32, np.float64
gamma = R.gamma


def _rel(a, b):
    return abs(float(a) - float(b)) / abs(float(b))


# ---------------------------------------------------------------------------------------------------------------- policies
def test_policies():
    assert R.scoremap_chunks(8, 256 * 256) == 33 and R.scoremap_chunks(1, 256) == 1 and R.scoremap_chunks(265, 289) == 1
    assert R.scoremap_chunks(13, 257) == 2 and R.scoremap_chunks(1, 65536) == 256
    assert R.reduction_blocks(2048) == (1, 2048) and R.reduction_blocks(2049) == (2, 1025)
    assert R.reduction_blocks(2 ** 21) == (1024, 2048) and R.reduction_blocks(2 ** 21 + 1) == (1024, 2049)
    assert R.reduction_blocks(3000001) == (1024, 2930)
    assert list(R.adam_chunk_prefix([0, 1, 8192, 8193])) == [0, 0, 1, 2, 4]
    per = R.adam_chunks_per_block([R.ADAM_CHUNK * 600])
    assert per.sum() == 600 and per.max() == 2 and per.min() == 1
    assert R.grid_for(1, 256) == 1 and R.grid_for(10 ** 9, 256) == 132 * 32
    assert R.resize_grad_passes(4, 4, 4, 4) == [] and [p for p, _ in R.resize_grad_passes(4, 5, 4, 6)] == ["cols"]


def test_fixed_sums_on_integers():
    """Integer-valued terms: every partial sum is exact, so each order gives the exact total"""
    rng = np.random.default_rng(1)
    for n in (1, 255, 256, 257, 1000, 70001):
        a = rng.integers(-50, 51, n).astype(f32)
        assert R.block_sum_fixed(a) == a.astype(f64).sum()
        nb, per = R.reduction_blocks(n)
        assert R.block_sum_fixed(R.blocked_sum(a, nb, per)) == a.astype(f64).sum()


def test_tree_is_the_kernels_pairing():
    """The tree adds red[t + h] into red[t] for h = 128 ... 1: three values that cancel only in that pairing"""
    red = np.zeros(256, f32)
    red[0], red[128], red[1] = 1.0, 2.0 ** 25, -(2.0 ** 25)
    # h = 128: red[0] = 1 + 2^25 (rounds to 2^25); ... h = 1: red[0] = 2^25 + (-2^25) = 0
    assert R.tree(red) == 0.0
    assert float(np.float64(1.0) + 2.0 ** 25 - 2.0 ** 25) == 1.0


# ---------------------------------------------------------------------------------------------------------------- resize gradient
RESIZE = [((3, 32, 32, 2), (256, 256)), ((2, 30, 17, 3), (97, 5)), ((1, 17, 23, 4), (5, 7)), ((2, 16, 12, 2), (16, 29)),
          ((2, 16, 12, 2), (7, 12)), ((1, 1, 1, 3), (7, 9)), ((2, 9, 11, 2), (1, 1)), ((1, 3, 1000, 1), (3, 3)),
          ((1, 3, 3, 1), (3, 1000)), ((2, 5, 3, 2), (5, 3))]


@pytest.mark.parametrize("shape,out", RESIZE, ids=lambda v: "x".join(map(str, v)))
def test_resize_grad_vs_fp64(shape, out):
    B, H, W, C = shape
    rng = np.random.default_rng(H * W + out[0])
    dy = rng.normal(size=(B, *out, C)).astype(f32)
    got = R.resize_grad(dy, H, W)
    ref = O.resize_bilinear_grad(dy, H, W)
    mag = O.resize_bilinear_grad(np.abs(dy), H, W)            # the weights are >= 0: the sum of |terms| of every output
    k = sum(2 * (R.cdiv(n_out, n_in) + 3) for n_in, n_out in ((W, out[1]), (H, out[0])) if n_in != n_out) + 2
    assert (np.abs(got - ref) <= gamma(k) * mag).all()
    if (H, W) == out:
        assert np.array_equal(got, dy)


def test_resize_grad_exact_on_integers_at_ratio_8():
    dy = np.random.default_rng(2).integers(-8, 9, size=(2, 64, 64, 3)).astype(f32)
    assert np.array_equal(R.resize_grad(dy, 8, 8), O.resize_bilinear_grad(dy, 8, 8))


def test_resize_grad_clamped_edge_takes_both_weights():
    """A 1-pixel input receives every output's two weights (i0 == i1 == 0): the total of dy, exactly for integers"""
    dy = np.arange(1, 8, dtype=f32).reshape(1, 7, 1, 1)
    assert R.resize_grad(dy, 1, 1)[0, 0, 0, 0] == 28.0


# ---------------------------------------------------------------------------------------------------------------- score-map loss
SCOREMAP = [(1, 1, 1), (1, 2, 3), (13, 10, 10), (8, 64, 64), (13, 1, 257), (300, 3, 4)]


@pytest.mark.parametrize("B,H,W", SCOREMAP, ids=lambda v: str(v))
def test_scoremap_loss_vs_fp64(B, H, W):
    rng = np.random.default_rng(B + H * W)
    P, T = rng.normal(size=(2, B, H, W, 21)).astype(f32)
    vis = rng.uniform(size=(B, 21)).astype(f32)
    vis[rng.uniform(size=(B, 21)) < 0.3] = 0
    loss, rms = R.scoremap_loss(P, T, vis)
    ref_loss, ref_rms = O.scoremap_loss(P, T, vis)
    e_rms, e_loss, e_grad = R.scoremap_bounds(B, H * W)
    assert (np.abs(rms - ref_rms) <= e_rms * ref_rms).all()
    assert _rel(loss, ref_loss) <= e_loss
    g = R.scoremap_loss_grad(P, T, vis, rms, -3.5)
    ref_g = O.scoremap_loss_grad(P, T, vis, -3.5)
    assert np.abs(g - ref_g).max() <= e_grad * np.abs(ref_g).max()


def test_scoremap_loss_exact_on_constant_differences():
    """P - T = +-c per map, small integers: rms = |c| exactly and the loss is f32(sum vis |c|) / f32(sum vis + 0.001)"""
    B, H, W = 13, 10, 10
    rng = np.random.default_rng(3)
    c = rng.integers(-5, 6, size=(B, 21)).astype(f32)
    T = rng.integers(-4, 5, size=(B, H, W, 21)).astype(f32)
    P = T + np.where(rng.uniform(size=(B, H, W, 21)) < 0.5, 1, -1).astype(f32) * c[:, None, None, :]
    vis = (rng.uniform(size=(B, 21)) < 0.7).astype(f32)
    loss, rms = R.scoremap_loss(P, T, vis)
    assert np.array_equal(rms, np.abs(c))
    assert loss == f32(f32((vis * np.abs(c)).astype(f64).sum()) / f32(f32(vis.astype(f64).sum()) + f32(0.001)))
    g = R.scoremap_loss_grad(P, T, vis, rms)
    assert not g.transpose(0, 3, 1, 2)[c == 0].any()           # rms == 0: no gradient


# ---------------------------------------------------------------------------------------------------------------- cross-entropy
@pytest.mark.parametrize("rows", [1, 255, 2049, 100003])
@pytest.mark.parametrize("labels", ["one_hot", "soft", "unnormalised"])
def test_xent_vs_fp64(rows, labels):
    rng = np.random.default_rng(rows)
    x = (rng.normal(size=(rows, 2)) * 4).astype(f32)
    x[3::7] *= 20
    if labels == "one_hot":
        h = rng.uniform(size=rows) < 0.3
        lab = np.stack([~h, h], 1).astype(f32)
    else:
        lab = rng.uniform(size=(rows, 2)).astype(f32)
        if labels == "soft":
            lab = (lab / lab.sum(1, keepdims=True)).astype(f32)
    nblk, per = R.xent_blocks(rows)
    k = R.cdiv(per, 256) + 8 + R.cdiv(nblk, 256) + 8 + 1
    # each row's value: log and exp within a few ulp, the row's two products and sums; the terms are all >= 0
    assert _rel(R.xent(x, lab), O.softmax_xent(x, lab)) <= gamma(k) + gamma(8)
    g = R.xent_grad(x, lab, 0.25)
    ref = O.softmax_xent_grad(x, lab, 0.25).reshape(-1, 2)
    assert np.abs(g - ref).max() <= gamma(8) * 0.25 / rows * (1 + np.abs(lab).max())


def test_xent_exact_canary():
    """logits (0, -200): exp(-200) is 0 in float32, s = 1, log s = 0, so each row gives exactly 200 label_1"""
    rows = 5000
    x = np.tile(np.array([0.0, -200.0], f32), (rows, 1))
    lab = np.zeros((rows, 2), f32)
    lab[::37, 1] = 1
    lab[::101, 1] = 2
    total = 200 * lab[:, 1].astype(f64).sum()
    assert R.xent(x, lab) == f32(f32(total) / f32(rows))


# ---------------------------------------------------------------------------------------------------------------- MSE
@pytest.mark.parametrize("n", [1, 255, 2049, 70001, 2 ** 21 + 1])
def test_mse_vs_fp64(n):
    rng = np.random.default_rng(n)
    p, q = rng.normal(size=(2, n)).astype(f32)
    nblk, per = R.mse_blocks(n)
    k = R.cdiv(per, 256) + 8 + R.cdiv(nblk, 256) + 8 + 3
    assert _rel(R.mse(p, q), L.mse(p, q)) <= gamma(k)
    ref = L.mse_grad(p, q, -2.5)
    assert np.abs(R.mse_grad(p, q, -2.5) - ref).max() <= gamma(3) * np.abs(ref).max()


def test_mse_exact_on_integers():
    rng = np.random.default_rng(4)
    n = 70001
    p = rng.integers(-5, 6, n).astype(f32)
    q = p + rng.integers(-3, 4, n).astype(f32)
    want = ((p.astype(f64) - q) ** 2).sum()
    assert want < 2 ** 24
    assert R.mse(p, q) == f32(f32(want) / f32(n))


# ---------------------------------------------------------------------------------------------------------------- Adam
def test_adam_restatement_is_within_fp64():
    """train_oracle.adam_tf_f32, which the GPU tables compare with bit for bit, against its fp64 form on the same float32 constants:
    each of p, m and v within a few roundings of its terms"""
    rng = np.random.default_rng(5)
    p, g = rng.normal(size=(2, 10000)).astype(f32)
    m, v = (rng.normal(size=10000) * 0.1).astype(f32), (rng.uniform(size=10000) * 0.01).astype(f32)
    b1p, b2p = O.beta_powers_after(3)
    c = dict(beta1=float(f32(0.9)), beta2=float(f32(0.999)), epsilon=float(f32(1e-8)))
    p1, m1, v1 = O.adam_tf_f32(p, g, m, v, f32(1e-3), b1p, b2p)
    p2, m2, v2 = O.adam_tf_f64(p, g, m, v, float(f32(1e-3)), float(b1p), float(b2p), **c)
    g64, m64, v64 = (a.astype(f64) for a in (g, m, v))
    assert (np.abs(m1 - m2) <= gamma(4) * (np.abs(m64) + np.abs(g64))).all()
    assert (np.abs(v1 - v2) <= gamma(4) * (v64 + g64 ** 2)).all()
    assert (np.abs(p1 - p2) <= gamma(16) * (np.abs(p) + np.abs(p2 - p))).all()

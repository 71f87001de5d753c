"""The dropout restatement (tests/dropout_oracle.py) on the host: its word layout against numpy's own Philox, keep_prob 1 as the
identity, the division-then-multiply order, the gradient's order and the keep fraction.  No GPU needed."""
import numpy as np
import pytest
from scipy import stats

import dropout_oracle as D

f32 = np.float32


@pytest.mark.parametrize("seed,draw,layer", [(0, 0, 0), (7, 3, 2), (2 ** 64 - 1, 12345, 4)])
def test_word_layout_matches_numpy_philox(seed, draw, layer):
    """Element (row, col) takes word col % 4 of the block at counter (draw, layer, row, col // 4) under key (seed, 2).  numpy's
    Philox increments its counter before it fills the buffer, so the block at counter c is what Philox(counter=c - 1) emits first."""
    rows, cols = 3, 10
    w = D.words(seed, draw, layer, rows, cols)
    key = np.array([seed, D.STREAM], np.uint64)
    for row in range(rows):
        for q in range((cols + 3) // 4):
            c = sum(v << (64 * j) for j, v in enumerate((draw, layer, row, q)))
            bg = np.random.Philox(key=int(key[0]) | (int(key[1]) << 64), counter=(c - 1) % 2 ** 256)
            block = bg.random_raw(4)
            for j in range(4):
                col = 4 * q + j
                if col < cols:
                    assert w[row, col] == block[j], (row, col)


def test_keep_prob_one_is_the_identity():
    x = np.random.default_rng(1).normal(size=(9, 37)).astype(f32) * f32(1e30)
    x[0, :4] = [0.0, -0.0, np.inf, -np.inf]
    y, k = D.dropout(x, 5, 0, 0, 1.0)
    assert (k == 1).all()
    assert np.array_equal(y.view(np.uint32), x.view(np.uint32))
    assert np.array_equal(D.backward(x, (k.astype(f32), 1.0)).view(np.uint32), x.view(np.uint32))


def test_division_then_multiplication():
    """x / 0.8f rounds differently from x * 1.25f for some fp32 x: the restatement divides, as TF does."""
    x = np.random.default_rng(2).uniform(-4, 4, size=100000).astype(f32)
    div = (x / f32(0.8)).astype(f32)
    mul = (x * f32(1.25)).astype(f32)
    assert (div != mul).any()
    ones = np.ones_like(x)
    assert np.array_equal(D.forward(x, (ones, 0.8)), div)
    # the gradient multiplies by the bit first, then divides: (dy * k) / keep_prob
    assert np.array_equal(D.backward(x, (ones, 0.8)), div)
    zeros = np.zeros_like(x)
    assert np.array_equal(np.signbit(D.forward(x, (zeros, 0.8))), np.signbit(x))


@pytest.mark.parametrize("keep_prob", [0.8, 0.75, 0.5])
def test_keep_fraction_within_binomial_bounds(keep_prob):
    rows, cols = 160, 512
    k = D.keep_bits(11, 4, 1, rows, cols, keep_prob)
    n = rows * cols
    lo, hi = stats.binom.ppf([1e-6, 1 - 1e-6], n, keep_prob)
    assert lo <= k.sum() <= hi, (k.sum(), lo, hi)
    # u is a multiple of 2^-24, so floor(keep_prob + u) keeps exactly the draws with u >= 1 - keep_prob (in fp32)
    u = D.uniform01(D.words(11, 4, 1, rows, cols))
    assert np.array_equal(k, (u >= f32(1) - f32(keep_prob)).astype(f32))


def test_seed_draw_layer_row_change_the_mask():
    base = D.keep_bits(3, 0, 0, 8, 128, 0.5)
    for args in ((4, 0, 0), (3, 1, 0), (3, 0, 1)):
        assert not np.array_equal(D.keep_bits(*args, 8, 128, 0.5), base), args
    assert not np.array_equal(base[0], base[1])


@pytest.mark.parametrize("half", [0, 1])
def test_planes_split_exactly(half):
    y = np.random.default_rng(3).normal(size=(5, 19)).astype(f32)
    hi, lo = D.planes(y, 64, half)
    assert hi.shape == (5, 64) and (hi[:, 19:] == 0).all() and (lo[:, 19:] == 0).all()
    if half == 1:
        back = hi.view(np.float16).astype(np.float64) + lo.view(np.float16).astype(np.float64)
    else:
        back = D._from_bf16(hi).astype(np.float64) + D._from_bf16(lo).astype(np.float64)
    assert np.abs(back[:, :19] - y).max() <= np.abs(y).max() * 2.0 ** -16

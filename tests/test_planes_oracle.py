"""Known answers for tests/planes_oracle.py, the numpy restatement of the activation plane formats that
test_gpu_conv_layer_planes.py holds the layer kernels to bit for bit.  CPU only."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import planes_oracle as P  # noqa: E402

f32, f64 = np.float32, np.float64


def _bits32(v):
    return np.asarray(v, f32).view(np.uint32)


def _bf16_rne_bits(v):
    """Bit-level round to nearest even of fp32 -> bf16 (finite inputs)."""
    u = _bits32(v).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def test_bf16_cast_equals_bit_level_rne():
    rng = np.random.default_rng(0)
    v = np.concatenate([rng.normal(size=20000) * np.exp2(rng.integers(-140, 120, size=20000)),
                        # every tie pattern: the 16 dropped bits exactly 0x8000, with even and odd kept mantissas
                        (_bits32(rng.normal(size=4000).astype(f32)) & np.uint32(0xFFFF0000) | np.uint32(0x8000)).view(f32)])
    v = v.astype(f32)
    v = v[np.isfinite(v) & (np.abs(v) < 3e38)]
    np.testing.assert_array_equal(P.bf16_bits(v), _bf16_rne_bits(v))


def test_bf16_ties_round_to_even():
    one_ulp = 2.0 ** -7   # bf16 spacing in [1, 2)
    v = np.array([1 + one_ulp / 2, 1 + 3 * one_ulp / 2, -(1 + one_ulp / 2), 1 + one_ulp / 2 + 2.0 ** -20], f32)
    np.testing.assert_array_equal(P.bf16_bits(v), np.array([0x3F80, 0x3F82, 0xBF80, 0x3F81], np.uint16))
    hi, lo = P.split16(v, "bf16")
    # lo carries the rounding: 1 + 3/2 ulp -> hi = 1 + 2 ulp, lo = -ulp / 2 = -2^-8
    assert lo[1] == 0xBB80 and P.bf16_value(lo[1]) == -(2.0 ** -8)
    np.testing.assert_array_equal(P.decode({"hi": hi, "lo": lo}, "bf16x3")[:3], v[:3].astype(f64))   # 2^-20 is past 16 bits


def test_fp16_ties_and_subnormal_lo():
    v = np.array([1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11], f32)   # half an fp16 ulp above 1 and above 1 + ulp
    np.testing.assert_array_equal(P.fp16_bits(v), np.array([0x3C00, 0x3C02], np.uint16))
    # 0.125 + 2^-20: hi = 0.125, lo = 2^-20 = 16 subnormal steps of 2^-24
    hi, lo = P.split16(np.array([0.125 + 2.0 ** -20], f32), "fp16")
    assert hi[0] == 0x3000 and lo[0] == 0x0010
    # lo below a subnormal step rounds: + 2^-26 (a quarter step) is dropped, + 2^-25 (half a step) ties to the even count 16,
    # + 3 2^-25 (one and a half steps) ties to 18
    for extra, code in ((2.0 ** -26, 0x0010), (2.0 ** -25, 0x0010), (3 * 2.0 ** -25, 0x0012)):
        hi, lo = P.split16(np.array([0.125 + 2.0 ** -20 + extra], f32), "fp16")
        assert hi[0] == 0x3000 and lo[0] == code, (extra, hex(int(lo[0])))
    # the smallest subnormal and its half (tie to zero)
    np.testing.assert_array_equal(P.fp16_bits(np.array([2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -25], f32)),
                                  np.array([0x0001, 0x0000, 0x0002], np.uint16))


def test_fp16_w_shift():
    colmax = np.array([1.0, 0.0, 2.0 ** -20, 3e38, 2.0 ** -149, np.nan, 0.75, 2.0 ** 14, -1.0], f32)
    np.testing.assert_array_equal(P.fp16_w_shift(colmax), [13, 0, 33, -114, 126, 0, 14, -1, 0])
    rng = np.random.default_rng(1)
    m = (np.abs(rng.normal(size=5000)) * np.exp2(rng.integers(-100, 100, size=5000))).astype(f32)
    m = m[m > 0]
    scaled = np.ldexp(m.astype(f64), P.fp16_w_shift(m))
    assert ((scaled >= 2.0 ** 13) & (scaled < 2.0 ** 14)).all()


def test_e4m3_saturation_and_subnormals():
    v = np.array([448, 449, 464, 1e6, np.inf, -448, -1e6, -np.inf, 2.0 ** -9, 2.0 ** -10, 3 * 2.0 ** -10, 2.0 ** -10 + 2.0 ** -20,
                  7 * 2.0 ** -9, 2.0 ** -6, 1.0, 0.25, 256.0, 0.0], f32)
    want = [0x7E, 0x7E, 0x7E, 0x7E, 0x7E, 0xFE, 0xFE, 0xFE, 0x01, 0x00, 0x02, 0x01, 0x07, 0x08, 0x38, 0x28, 0x78, 0x00]
    np.testing.assert_array_equal(P.e4m3_bits(v), np.array(want, np.uint8))
    codes = np.array([c for c in range(256) if c not in (0x7F, 0xFF)], np.uint8)   # every finite code decodes and re-encodes to itself
    np.testing.assert_array_equal(P.e4m3_bits(P.e4m3_value(codes)), codes)
    assert P.e4m3_value(np.array([0x7E, 0x01, 0x08], np.uint8)).tolist() == [448.0, 2.0 ** -9, 2.0 ** -6]


def test_f8c_known_answers():
    # v, h16, l8, h8, decoded
    cases = [(1.0, 0x5000, 0x00, 0x28, 1.0),
             (1 + 2.0 ** -12, 0x5000, 0x28, 0x28, 1 + 2.0 ** -12),                  # the residual 2^-12 is l8 = 0.25
             (2047.0, 0x7BFF, 0x00, 0x7E, 2047.0),                                  # main plane at its largest finite value
             (2047.25, 0x7BFF, 0x78, 0x7E, 2047.25),                                # 32 v = 65512 saturates; residual 256 is exact
             (2047.5, 0x7BFF, 0x7E, 0x7E, 2047.0 + 448 / 1024.0),                   # residual 512 saturates at 448
             (2046.5, 0x7BFE, 0x7E, 0x7E, 2046.0 + 448 / 1024.0),                   # 32 v = 65488 ties down to 65472 (even)
             (-2047.5, 0xFBFF, 0xFE, 0xFE, -(2047.0 + 448 / 1024.0)),
             (1e5, 0x7BFF, 0x7E, 0x7E, 2047.0 + 448 / 1024.0)]
    v = np.array([c[0] for c in cases], f32)
    h16, l8, h8 = P.f8c_planes(v)
    assert [int(x) for x in h16] == [c[1] for c in cases]
    assert [int(x) for x in l8] == [c[2] for c in cases]
    assert [int(x) for x in h8] == [c[3] for c in cases]
    np.testing.assert_array_equal(P.f8c_value(h16, l8), [c[4] for c in cases])
    # the clamp ignores NaN as fminf / fmaxf do
    assert P.f8c_planes(np.array([np.nan], f32))[0][0] == P.fp16_bits(np.array([-65504.0], f32))[0]


@pytest.mark.parametrize("prec", list(P.PLANES))
def test_round_trip(prec):
    """decode(encode(v)) is v within the format's resolution, across the binades the mode is documented for."""
    rng = np.random.default_rng(2)
    lo_e, hi_e = {"fp16_f8c": (-2, 10), "fp16x3": (-6, 14), "fp16": (-6, 14)}.get(prec, (-30, 30))
    v = (rng.normal(size=50000) * np.exp2(rng.integers(lo_e, hi_e, size=50000))).astype(f32)
    if prec == "fp16_f8c":
        v = np.clip(v, -2000, 2000)
    planes = P.encode(v, prec)
    assert set(planes) == set(P.PLANES[prec])
    err = np.abs(P.decode(planes, prec) - v.astype(f64))
    assert (err <= P.FORMAT_REL[prec] * np.abs(v) + P.FORMAT_ABS[prec]).all(), prec


@pytest.mark.parametrize("half", ["bf16", "fp16"])
def test_split_invariant(half):
    """Every split satisfies split_ok, including just below the powers of two (half the spacing below them) and the ties; a lo
    written from v instead of v - hi does not."""
    rng = np.random.default_rng(3)
    v = (rng.normal(size=50000) * np.exp2(rng.integers(-6, 12, size=50000))).astype(f32)
    v = np.concatenate([v, np.exp2(np.arange(-6, 12)).astype(f32) * f32(1 - 2.0 ** -20), np.float32([0.0, -0.0])])
    hi, lo = P.split16(v, half)
    assert P.split_ok(hi, lo, half).all()
    # hi = rn16(hi + lo) holds except at the midpoints, which are rare but do occur among 50000 draws
    ties = P.ENC16[half]((P.DEC16[half](hi).astype(f64) + P.DEC16[half](lo)).astype(f32)) != hi
    assert 0 < ties.sum() < 200
    assert not P.split_ok(hi, P.ENC16[half](v), half)[v != 0].any()

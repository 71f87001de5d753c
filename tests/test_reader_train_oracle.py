"""CPU pins of the RHD reader's training mode (tests/reader_train_oracle.py): the Philox restatement against numpy.random.Philox,
the distributions of the parameter generator (fixed seeds, so deterministic), TF 1.3 adjust_hue against TensorFlow's own test
tables and colorsys, the steady-state shuffle queue, and the sample restatement against the vectors the reference's unmodified reader
produced with scripted draws (golden_reference_reader_train.npz)."""
import colorsys
import os
import sys

import numpy as np
import pytest
from scipy import stats

import reader_train_oracle as A

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_reference_reader_train as MT  # noqa: E402
import synth_records as SR  # noqa: E402
from oracle import reader_oracle as R  # noqa: E402

f32 = np.float32
G = np.load(os.path.join(HERE, "golden", "golden_reference_reader_train.npz"))


# ------------------------------------------------------------------------------------------ generator
def _minus_one(ctr):
    n = sum(int(c) << (64 * i) for i, c in enumerate(ctr))
    n = (n - 1) % (1 << 256)
    return np.array([(n >> (64 * i)) & A.M64 for i in range(4)], np.uint64)


@pytest.mark.parametrize("ctr,key", [([0, 0, 0, 0], [0, 0]), ([1, 0, 0, 0], [5, 1]), ([0, 1, 0, 0], [2 ** 64 - 1, 0]),
                                     ([0, 0, 1, 0], [123456789, 1]), ([0, 0, 0, 1], [7, 7]), ([2 ** 64 - 1, 2 ** 64 - 1, 3, 0], [1, 2]),
                                     ([41257, 84, 15, 0], [20171003, 0])])
def test_philox_matches_numpy_across_carries(ctr, key):
    """numpy.random.Philox pre-increments its 256-bit counter (with carry), so counter = c - 1 yields Philox(c, key) first."""
    ref = np.random.Philox(counter=_minus_one(ctr), key=np.array(key, np.uint64)).random_raw(4)
    got = A.philox4x64_10(np.array([ctr], np.uint64), np.array([key], np.uint64))[0]
    np.testing.assert_array_equal(got, ref)


def test_shuffle_stream_is_numpy_philox_from_counter_zero():
    ref = np.random.Philox(key=np.array([99, A.STREAM_SHUFFLE], np.uint64)).random_raw(37)
    np.testing.assert_array_equal(A.shuffle_words(99, 37), ref)


def test_truncated_normal_distribution():
    z, att = A.truncated_normal(11, np.arange(20000), 5, return_attempts=True)
    assert np.abs(z).max() <= 2.0
    assert stats.kstest(z.astype(np.float64), stats.truncnorm(-2, 2).cdf).pvalue > 0.01
    assert att.min() == 0 and (att >= 1).mean() < 0.01          # both draws of an attempt rejected: ~0.2 %
    assert not np.array_equal(z, A.truncated_normal(12, np.arange(20000), 5))
    p = A.aug_params(3, np.arange(2000), A.COORD_UV_NOISE | A.CROP_CENTER_NOISE | A.CROP_OFFSET_NOISE)
    for sl, sigma in ((slice(0, 84), 2.5), (slice(84, 86), 20.0), (slice(87, 89), 10.0)):
        v = p[:, sl]
        assert np.abs(v).max() <= 2 * sigma and abs(v.std() / sigma - stats.truncnorm(-2, 2).std()) < 0.03
        np.testing.assert_array_equal(v[:, 0], (A.truncated_normal(3, np.arange(2000), sl.start) * f32(sigma)).astype(f32))


def test_uniform_ranges_and_tf_affine_step():
    assert f32(1.2) - f32(1.0) == f32(0.20000005)                 # TF computes maxval - minval in fp32
    u = A.uniform01(A.words(1, np.arange(50000), A.SCALE)[:, 0])
    assert u.min() >= 0 and u.max() < 1 and np.all(u * f32(2 ** 24) == np.floor(u * f32(2 ** 24)))
    p = A.aug_params(1, np.arange(50000), A.CROP_SCALE_NOISE | A.HUE)
    s, h = p[:, A.SCALE], p[:, A.HUE_DELTA]
    np.testing.assert_array_equal(s, (u * f32(0.20000005) + f32(1.0)).astype(f32))
    assert s.min() >= 1.0 and s.max() < f32(1.2) and abs(float(s.mean()) - 1.1) < 2e-3
    assert h.min() >= f32(-0.1) and h.max() < f32(0.1) and abs(float(h.mean())) < 2e-3
    assert stats.kstest(s.astype(np.float64), stats.uniform(1.0, 0.2).cdf).pvalue > 0.01


def test_window_offsets_chi_square():
    p = A.aug_params(4, np.arange(65 * 300), A.RANDOM_CROP)
    for j in (A.WINDOW, A.WINDOW + 1):
        o = p[:, j].astype(np.int64)
        assert o.min() == 0 and o.max() == 64 and np.all(p[:, j] == o)
        assert stats.chisquare(np.bincount(o, minlength=65)).pvalue > 1e-3
    assert stats.pearsonr(p[:, A.WINDOW], p[:, A.WINDOW + 1])[0] < 0.05


def test_keep_rate():
    p = A.aug_params(6, np.arange(20000), A.SCOREMAP_DROPOUT)
    k = p[:, A.KEEP:A.KEEP + 21]
    assert set(np.unique(k)) == {0.0, 1.0}
    assert abs(k.mean() - 0.8) < 4 * np.sqrt(0.16 / k.size)
    u = A.uniform01(A.words(6, np.arange(20000), A.KEEP)[:, 0])
    np.testing.assert_array_equal(k[:, 0], np.floor(f32(0.8) + u))      # floor(keep_prob + u) in fp32, as TF 1.3's dropout


def test_flags_off_params_are_neutral():
    p = A.aug_params(8, np.arange(16), 0)
    assert np.all(p[:, A.SCALE] == 1) and np.all(p[:, A.KEEP:A.KEEP + 21] == 1)
    assert np.all(np.delete(p, [A.SCALE] + list(range(A.KEEP, A.KEEP + 21)), 1) == 0)
    full = A.aug_params(8, np.arange(16), 127)
    for flags in (A.COORD_UV_NOISE, A.HUE, A.SCOREMAP_DROPOUT):   # a value depends on (seed, serial, slot), not on the other flags
        one = A.aug_params(8, np.arange(16), flags)
        on = np.any(one != p, 0)
        np.testing.assert_array_equal(one[:, on], full[:, on])


# ------------------------------------------------------------------------------------------ adjust_hue
def test_adjust_hue_tf_tables():
    """image_ops_test.py AdjustHueTest.testAdjustNegativeHue / testAdjustPositiveHue (uint8 in, convert_image_dtype both ways)."""
    x = np.array([0, 5, 13, 54, 135, 226, 37, 8, 234, 90, 255, 1], np.uint8).reshape(2, 2, 3)
    for delta, y in ((-0.25, [0, 13, 1, 54, 226, 59, 8, 234, 150, 255, 39, 1]), (0.25, [13, 0, 11, 226, 54, 221, 234, 8, 92, 1, 217, 255])):
        o = A.adjust_hue(x.astype(f32) * f32(1.0 / 255.0), f32(delta))
        np.testing.assert_array_equal((o * f32(255.5)).astype(np.uint8).reshape(-1), y)


def test_hsv_against_colorsys_in_range():
    rng = np.random.default_rng(0)
    rgb = rng.uniform(0, 1, size=(500, 3)).astype(f32)
    rgb[:20] = rgb[:20, :1]                                     # grey pixels: range 0
    hsv = A.rgb_to_hsv(rgb)
    for i in range(rgb.shape[0]):
        np.testing.assert_allclose(hsv[i], colorsys.rgb_to_hsv(*rgb[i].astype(np.float64)), atol=2e-6)
        np.testing.assert_allclose(A.hsv_to_rgb(hsv[i]), colorsys.hsv_to_rgb(*hsv[i].astype(np.float64)), atol=2e-6)
    for delta in (-0.1, -0.03, 0.05, 0.0999):
        o = A.adjust_hue(rgb, f32(delta))
        for i in range(0, rgb.shape[0], 7):
            h, s, v = colorsys.rgb_to_hsv(*rgb[i].astype(np.float64))
            np.testing.assert_allclose(o[i], colorsys.hsv_to_rgb((h + delta + 1.0) % 1.0, s, v), atol=5e-6)


def test_adjust_hue_grey_collapse_on_non_positive_max():
    """S = V > 0 ? range / V : 0: a pixel whose largest channel is <= 0 comes back as (V, V, V) -- the dark half of image / 255 - 0.5."""
    px = np.array([[-0.5, -0.2, -0.3], [-0.1, -0.4, 0.0], [-0.49, -0.5, -0.01], [0.3, -0.2, -0.4]], f32)
    o = A.adjust_hue(px, f32(0.07))
    v = px.max(1)
    np.testing.assert_array_equal(o[:3], np.repeat(v[:3, None], 3, 1))
    assert not np.all(o[3] == o[3, 0])                           # V > 0 with negative channels: S > 1, still a hue rotation


# ------------------------------------------------------------------------------------------ shuffle queue
def test_shuffle_queue_order():
    s = A.shuffle_serials(13, 20000)
    d = np.arange(s.size)
    assert np.all(s < d + 100)                                    # nothing is dequeued before it is enqueued
    assert np.unique(s).size == s.size                            # nor twice
    late = s >= 100                                               # serial k >= 100 enters the buffer after dequeue k - 100
    age = d[late] - (s[late] - 100) - 1
    assert age.min() >= 0
    np.testing.assert_allclose(age.mean(), 99.0, rtol=0.05)       # steady state: Geometric(1 / 100) on {0, 1, ...}
    cnt = np.bincount(np.minimum(age, 400) // 20, minlength=21)[:21]
    edges = np.arange(0, 421, 20)
    pr = 0.99 ** edges[:-1] - 0.99 ** edges[1:]
    pr[-1] = 0.99 ** 400
    assert stats.chisquare(cnt, pr / pr.sum() * cnt.sum()).pvalue > 1e-3
    np.testing.assert_array_equal(s, A.shuffle_serials(13, 20000))
    assert not np.array_equal(s[:200], A.shuffle_serials(14, 200))


def test_reader_queue_matches_restatement_for_any_batch_size():
    from hand3d_b200.data.BinaryDbReader import _ShuffleQueue
    ref = A.shuffle_serials(21, 96)
    for bs in (1, 8, 32, 96):
        q = _ShuffleQueue(21)
        np.testing.assert_array_equal(np.concatenate([q.take(bs) for _ in range(96 // bs)]), ref)


# ------------------------------------------------------------------------------------------ against the reference reader
def _cfg(name):
    kw = dict(MT.CONFIGS[name])
    kw.pop("shuffle")
    return A.flags_of(**kw), {k: kw[k] for k in ("use_wrist_coord", "hand_crop") if k in kw}


@pytest.mark.parametrize("name", list(MT.CONFIGS))
def test_oracle_against_reference_golden(name):
    recs = SR.rhd_records(4)
    flags, kw = _cfg(name)
    seed = int(G["seed"])
    params = A.aug_params(seed, G["serials"], flags)
    for i in range(4):
        pre = "%s/%d/" % (name, i)
        np.testing.assert_array_equal(G[pre + "params"], params[i])
        d = A.rhd_items_train(recs[i], params[i], flags, **kw)
        keys = sorted({k.split("/")[2] for k in G.files if k.startswith(pre)} - {"params", "calls"})
        assert keys == sorted(set(d) - {"crop_center"}), (keys, sorted(d))
        for k in keys:
            v = np.asarray(d[k])
            if pre + k + "/sub8" in G.files:
                np.testing.assert_array_equal(v.shape, G[pre + k + "/shape"])
                np.testing.assert_allclose(v[::8, ::8], G[pre + k + "/sub8"], atol=1e-6, err_msg=k)
                np.testing.assert_allclose([v.astype(np.float64).sum(), np.square(v.astype(np.float64)).sum()], G[pre + k + "/sums"],
                                           rtol=1e-6, atol=1e-6, err_msg=k)
            else:
                np.testing.assert_allclose(v.astype(np.float64), G[pre + k].astype(np.float64), atol=1e-6, rtol=1e-6, err_msg=k)
        calls = set(G[pre + "calls"].tolist())
        assert ("random_hue" in calls) == bool(flags & A.HUE) and ("dropout" in calls) == bool(flags & A.SCOREMAP_DROPOUT)
        assert ("random_crop" in calls) == bool(flags & A.RANDOM_CROP) and "shuffle_batch_join" in calls
    if flags & A.SCOREMAP_DROPOUT:
        assert (params[:, A.KEEP:A.KEEP + 21] == 0).any()           # the golden covers dropped channels


@pytest.mark.parametrize("kw", [dict(use_wrist_coord=False, hand_crop=True), dict(use_wrist_coord=True), dict(scale_to_size=True)])
def test_flags_off_equals_evaluation_oracle(kw):
    recs = SR.rhd_records(4)
    neutral = A.aug_params(0, [0], 0)[0]
    for i in range(4):
        ref, d = R.rhd_items(recs[i], **kw), A.rhd_items_train(recs[i], neutral, 0, **kw)
        for k in d:
            np.testing.assert_array_equal(np.asarray(d[k]), np.asarray(ref[k]), err_msg=k)

"""The numpy restatement of the device evaluator (tests/eval_oracle.py) against numpy itself, bit for bit, and DeviceEvalUtil's host
finish (measures_from_stats) against the reference-API EvalUtil fed sample by sample.  No GPU needed."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import eval_oracle as EO
from hand3d_b200 import _lib
from hand3d_b200.utils.general import EvalUtil, measures_from_stats

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, "tests", "golden", "golden_reference_numpy.npz"))
SIZES = list(range(1, 300)) + [1000, 2728, 8191, 8192, 8193, 9000, 20000, 41258]


def _values(rng, n, dtype):
    return (2.0 ** rng.uniform(-20, 20, n)).astype(dtype)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_pairwise_mean_equals_numpy(dtype):
    rng = np.random.default_rng(11)
    for n in SIZES:
        a = _values(rng, n, dtype)
        m = EO.mean(a)
        assert m.dtype == dtype and m == np.mean(a), n
        assert EO.pairwise_sum(a) == np.sum(a), n


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_pairwise_mean_equals_numpy_at_a_million(dtype):
    a = _values(np.random.default_rng(12), 10 ** 6, dtype)
    assert EO.mean(a) == np.mean(a)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_median_equals_numpy(dtype):
    rng = np.random.default_rng(13)
    for n in SIZES + [10 ** 6]:
        a = _values(rng, n, dtype)
        m = EO.median(a)
        assert m.dtype == dtype and m == np.median(a), n


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_ties_zeros_inf_and_nan(dtype):
    rng = np.random.default_rng(14)
    for n in (1, 2, 7, 8, 9, 128, 129, 130, 1000, 2728):
        base = rng.choice(np.array([0.0, 1.0, 2.0, 3.0, 2.0 ** -20, 2.0 ** 20], dtype), n)
        for a in (base, np.where(rng.uniform(size=n) < 0.1, dtype(np.inf), base), np.where(rng.uniform(size=n) < 0.1, dtype(np.nan), base)):
            a = a.astype(dtype)
            np.testing.assert_array_equal(EO.mean(a), np.mean(a))
            np.testing.assert_array_equal(EO.median(a), np.median(a))
            thr = np.linspace(0.0, 3.0, 20)
            np.testing.assert_array_equal(EO.counts(a, thr), [np.count_nonzero(a <= t) for t in thr])


def test_frontier_fits_the_device_buffer():
    """csrc/eval.cu cuts pairwise_sum's tree into at most kFrontier = 1024 subtrees for every n up to 2^24."""
    worst = max(EO.frontier_nodes(n) for n in list(range(1, 5000)) + list(range(5000, 1 << 24, 9973)) + [1 << 24])
    assert worst <= 1024


def _feed_all(ev, tag):
    for i in range(G[tag + "_gt"].shape[0]):
        ev.feed(G[tag + "_gt"][i], G[tag + "_vis"][i], G[tag + "_pred"][i])


@pytest.mark.parametrize("tag", ["ev2", "ev3"])
@pytest.mark.parametrize("steps", [1, 2, 20, 100])
def test_measures_from_stats_equal_evalutil(tag, steps):
    ev = EvalUtil()
    _feed_all(ev, tag)
    lists = EO.feed_lists(G[tag + "_gt"], G[tag + "_vis"], G[tag + "_pred"])
    for k in range(21):
        np.testing.assert_array_equal(lists[k], np.array(ev.data[k], dtype=np.float64))
    lo, hi, _ = G[tag + "_range"]
    with np.errstate(invalid="ignore", divide="ignore"):
        want = ev.get_measures(float(lo), float(hi), steps)
        got = measures_from_stats(EO.stats(lists, np.linspace(float(lo), float(hi), steps)), float(lo), float(hi), steps, np.float64)
    for w, g in zip(want, got):
        assert np.asarray(g).dtype == np.asarray(w).dtype
        np.testing.assert_array_equal(g, w)
    if tag == "ev2":
        assert len(lists[13]) == 0          # the key-point that is never visible


@pytest.mark.parametrize("tag", ["ev2", "ev3"])
def test_degenerate_range_gives_nan_on_both(tag):
    ev = EvalUtil()
    _feed_all(ev, tag)
    lists = EO.feed_lists(G[tag + "_gt"], G[tag + "_vis"], G[tag + "_pred"])
    with np.errstate(invalid="ignore", divide="ignore"):
        want = ev.get_measures(5.0, 5.0, 20)
        got = measures_from_stats(EO.stats(lists, np.linspace(5.0, 5.0, 20)), 5.0, 5.0, 20, np.float64)
    assert np.isnan(want[2]) and np.isnan(got[2])
    for w, g in zip(want, got):
        np.testing.assert_array_equal(g, w)


def test_float32_measures_from_stats_equal_evalutil():
    rng = np.random.default_rng(15)
    gt = rng.normal(size=(300, 21, 3)).astype(np.float32)
    pred = (gt + rng.normal(scale=0.02, size=gt.shape)).astype(np.float32)
    vis = rng.uniform(size=(300, 21)) > 0.3
    vis[:, 4] = False
    ev = EvalUtil()
    for i in range(300):
        ev.feed(gt[i], vis[i], pred[i])
    lists = EO.feed_lists(gt, vis, pred)
    assert lists[0].dtype == np.float32
    with np.errstate(invalid="ignore"):
        want = ev.get_measures(0.0, 0.05, 20)
        got = measures_from_stats(EO.stats(lists, np.linspace(0.0, 0.05, 20)), 0.0, 0.05, 20, np.float32)
    for w, g in zip(want, got):
        assert np.asarray(g).dtype == np.asarray(w).dtype
        np.testing.assert_array_equal(g, w)


# ------------------------------------------------------------------------------------------- C ABI (no device needed)
def test_eval_symbols_declared_exported_and_bound():
    hdr = open(os.path.join(ROOT, "include", "hand3d_b200.h")).read()
    lib = _lib.load()
    assert lib.h3d_version() >= 105
    for name in ("h3d_eval_store_bytes", "h3d_eval_feed", "h3d_eval_stats"):
        assert re.search(r"H3D_API\s+[\w\s\*]+?\b%s\s*\(" % name, hdr), name
        assert name in _lib.SIGNATURES
        getattr(lib, name)
    for macro, value in (("H3D_EVAL_FLOAT32", _lib.EVAL_FLOAT32), ("H3D_EVAL_FLOAT64", _lib.EVAL_FLOAT64), ("H3D_EVAL_KEPT", _lib.EVAL_KEPT),
                         ("H3D_EVAL_DROPPED", _lib.EVAL_DROPPED), ("H3D_EVAL_TICKET", _lib.EVAL_TICKET), ("H3D_EVAL_COUNT", _lib.EVAL_COUNT),
                         ("H3D_EVAL_HEADER_WORDS", _lib.EVAL_HEADER_WORDS), ("H3D_EVAL_MAX_KP", _lib.EVAL_MAX_KP),
                         ("H3D_EVAL_MAX_DIM", _lib.EVAL_MAX_DIM), ("H3D_EVAL_MAX_SAMPLES", _lib.EVAL_MAX_SAMPLES),
                         ("H3D_EVAL_MAX_THRESHOLDS", _lib.EVAL_MAX_THRESHOLDS), ("H3D_EVAL_STAT_N", _lib.EVAL_STAT_N),
                         ("H3D_EVAL_STAT_MEAN", _lib.EVAL_STAT_MEAN), ("H3D_EVAL_STAT_MEDIAN", _lib.EVAL_STAT_MEDIAN),
                         ("H3D_EVAL_STAT_COUNTS", _lib.EVAL_STAT_COUNTS)):
        assert int(re.search(r"#define %s (\d+)" % macro, hdr).group(1)) == value, macro
    assert _lib.EVAL_COUNT + _lib.EVAL_MAX_KP <= _lib.EVAL_HEADER_WORDS
    from utils.general import DeviceEvalUtil as shim
    from hand3d_b200.utils.general import DeviceEvalUtil
    assert shim is DeviceEvalUtil


def test_store_bytes():
    lib = _lib.load()
    h = _lib.EVAL_HEADER_WORDS * 8
    assert lib.h3d_eval_store_bytes(21, 2728, _lib.EVAL_FLOAT32) == h + 21 * 2728 * 4
    assert lib.h3d_eval_store_bytes(21, 2728, _lib.EVAL_FLOAT64) == h + 21 * 2728 * 8
    assert lib.h3d_eval_store_bytes(64, 1 << 24, _lib.EVAL_FLOAT64) == h + 64 * (1 << 24) * 8


BAD_STORES = [(0, 10, 0), (65, 10, 0), (21, 0, 0), (21, (1 << 24) + 1, 1), (21, 10, 2), (21, 10, -1)]


@pytest.mark.parametrize("K,N,dtype", BAD_STORES)
def test_limits_are_refused(K, N, dtype):
    lib = _lib.load()
    assert lib.h3d_eval_store_bytes(K, N, dtype) == _lib.EINVAL
    p = C.c_void_p(8)      # never dereferenced: the limits are checked first
    assert lib.h3d_eval_feed(None, p, K, N, dtype, p, p, p, 1, 2, None) == _lib.EINVAL
    msg = _lib.last_error()
    assert "h3d_eval_feed" in msg and ("K =" in msg or "num_samples" in msg or "dtype" in msg), msg
    assert lib.h3d_eval_stats(None, p, K, N, dtype, p, 20, p, None) == _lib.EINVAL
    assert "h3d_eval_stats" in _lib.last_error()


@pytest.mark.parametrize("D", [0, 5])
def test_dimension_limit_is_refused(D):
    lib = _lib.load()
    p = C.c_void_p(8)
    assert lib.h3d_eval_feed(None, p, 21, 10, 0, p, p, p, 1, D, None) == _lib.EINVAL
    assert "D = %d" % D in _lib.last_error()


@pytest.mark.parametrize("T", [0, 4097])
def test_threshold_limit_is_refused(T):
    lib = _lib.load()
    p = C.c_void_p(8)
    assert lib.h3d_eval_stats(None, p, 21, 10, 0, p, T, p, None) == _lib.EINVAL
    assert "T = %d" % T in _lib.last_error()


def test_host_side_limits_are_refused():
    from hand3d_b200.utils.general import DeviceEvalUtil
    with pytest.raises(TypeError):
        DeviceEvalUtil(21)
    for kw in ({"num_kp": 0, "num_samples": 5}, {"num_kp": 65, "num_samples": 5}, {"num_kp": 21, "num_samples": 0},
               {"num_kp": 21, "num_samples": (1 << 24) + 1}):
        with pytest.raises(ValueError):
            DeviceEvalUtil(**kw)

"""The tracking rule's numpy restatement (tests/track_oracle.py) on hand-worked cases: the next crop from key-points, both scale clamps,
a zero-size box, the fall-backs for non-finite key-points, the score and when a slot is lost."""
import numpy as np

import track_oracle as T

F = np.float32


def _uv(points, rest=(128, 128)):
    uv = np.tile(np.array(rest, np.int32), (21, 1))
    for k, p in enumerate(points):
        uv[k] = p
    return uv


def _map(peak, B=1):
    m = np.full((B, 32, 32, 21), F(peak) - F(1), F)
    m[:, 3, 4, :] = peak
    return m


def test_crop_without_clamp():
    # rows (64-128)/2+120 = 88 .. (192-128)/2+120 = 152, cols (64-128)/2+160 = 128 .. (160-128)/2+160 = 176
    c, s, fb = T.next_crop(_uv([(64, 64), (192, 160)]), (120, 160), 2.0, 1.5)
    np.testing.assert_array_equal(c, F([120, 152]))
    assert s == F(256) / F(96) and not fb                          # size 64 rows, x 1.5


def test_crop_upper_clamp():
    # rows 192 .. 208 (extent 16), cols 292 .. 302 (extent 10): 256 / 24 > 5
    c, s, fb = T.next_crop(_uv([(120, 120), (136, 130)]), (200, 300), 1.0, 1.5)
    np.testing.assert_array_equal(c, F([200, 297]))
    assert s == F(5.0) and not fb


def test_crop_lower_clamp():
    # rows -412 .. 608 (extent 1020), cols -312 .. 200: 256 / 1530 < 0.25
    c, s, fb = T.next_crop(_uv([(0, 0), (255, 100)]), (100, 200), 0.25, 1.5)
    np.testing.assert_array_equal(c, F([98, -56]))
    assert s == F(0.25) and not fb


def test_all_keypoints_on_one_pixel():
    uv = np.tile(np.array([50, 60], np.int32), (21, 1))
    c, s, fb = T.next_crop(uv, (100, 100), 2.0, 1.5)
    np.testing.assert_array_equal(c, F([61, 66]))                  # (50-128)/2+100, (60-128)/2+100
    assert s == F(5.0) and not fb                                  # size 0: 256 / 0 = inf, clamped


def test_margin_is_applied():
    _, s125, _ = T.next_crop(_uv([(64, 64), (192, 160)]), (120, 160), 2.0, 1.25)
    assert s125 == F(256) / (F(64) * F(1.25))


def test_non_finite_inputs_fall_back_and_are_lost():
    state = T.new_state(4)
    state["center"][:] = [[10, 20], [30, 40], [50, 60], [70, 80]]
    state["scale"][:] = [1, 2, 3, 4]
    before = {k: v.copy() for k, v in state.items()}
    uv = np.stack([_uv([(0, 0), (255, 255)])] * 4)
    center = F([[100, 100], [np.nan, 100], [100, np.inf], [100, 100]])
    scale = F([0.0, 1.0, 1.0, np.nan])                             # x / 0 -> inf (and 0 / 0 -> NaN at uv 128)
    for b in range(3):
        c, s, fb = T.next_crop(uv[b], center[b], scale[b], 1.5)
        assert fb
        np.testing.assert_array_equal(c, F([160, 160]))
        assert s == F(256) / (F(100) * F(1.5))
    T.update(state, _map(1.0, 4), uv, center, scale, 1.5, min_score=None)
    np.testing.assert_array_equal(state["lost"], [1, 1, 1, 1])
    np.testing.assert_array_equal(state["center"], before["center"])  # a lost slot keeps its crop
    np.testing.assert_array_equal(state["scale"], before["scale"])
    np.testing.assert_array_equal(state["score"], F([1, 1, 1, 1]))


def test_score_is_the_mean_peak():
    m = np.zeros((32, 32, 21), F)
    for k in range(21):
        m[k % 32, (3 * k) % 32, k] = F(k + 1) / F(8)
    m[5, 5, 0] = F(-3)                                             # not a peak
    want = F(0)
    for k in range(21):
        want = F(want + F(k + 1) / F(8))
    assert T.score(m) == F(want / F(21))
    assert np.isnan(T.score(np.where(np.arange(32 * 32 * 21).reshape(32, 32, 21) == 777, np.nan, m).astype(F)))
    assert np.signbit(T.score(np.full((32, 32, 21), -0.0, F))) == False   # the sum starts from +0


def test_nan_score_is_lost_only_with_min_score():
    uv = _uv([(64, 64), (192, 160)])[None]
    nan_map = _map(1.0)
    nan_map[0, 5, 5, 7] = np.nan
    for min_score, lost in ((None, 0), (0.5, 1), (-1e30, 1)):
        st = T.new_state(1)
        T.update(st, nan_map, uv, F([[120, 160]]), F([2.0]), 1.5, min_score=min_score)
        assert np.isnan(st["score"][0]) and st["lost"][0] == lost, min_score
        if not lost:
            np.testing.assert_array_equal(st["center"][0], F([120, 152]))


def test_min_score_threshold():
    uv = _uv([(64, 64), (192, 160)])[None]
    for peak, min_score, lost in ((0.5, 0.5, 0), (0.5, 0.5000001, 1), (0.0, None, 0), (-5.0, None, 0), (2.0, 1.0, 0)):
        st = T.new_state(1)
        T.update(st, _map(peak), uv, F([[120, 160]]), F([2.0]), 1.5, min_score=min_score)
        assert st["score"][0] == F(peak) and st["lost"][0] == lost, (peak, min_score)
        if lost:
            np.testing.assert_array_equal(st["center"][0], T.new_state(1)["center"][0])
        else:
            assert st["scale"][0] == F(256) / F(96)

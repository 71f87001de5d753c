"""The drawing rule of h3d_draw_segments (tests/draw_oracle.py), worked by hand on small images: full and half coverage, round caps,
discs, non-finite and off-image segments, painting order, valid, and the palette's .5 entries."""
import numpy as np
import pytest

import draw_oracle as O
from hand3d_b200 import draw as D

F = np.float32
C = np.float32([[200.0, 100.0, 50.0]])


def _blank(H=32, W=40, v=0):
    return np.full((1, H, W, 3), v, np.uint8)


def _one(seg, lw=1.0, colors=C, img=None, valid=None):
    img = _blank() if img is None else img
    return O.draw(img, np.float32(seg).reshape(1, -1, 4), colors, lw, valid)[0]


def test_linewidth_1_on_a_pixel_row():
    out = _one([10.0, 5.0, 10.0, 20.0])
    np.testing.assert_array_equal(out[10, 5:21], np.repeat(np.uint8([[200, 100, 50]]), 16, 0))
    assert not out[9].any() and not out[11].any()
    assert not out[10, :4].any() and not out[10, 22:].any()     # one pixel past either end: d = 1, a = 0 at h = 1


def test_between_two_rows_half_each():
    out = _one([10.5, 5.0, 10.5, 20.0])
    for r in (10, 11):
        np.testing.assert_array_equal(out[r, 5:21], np.repeat(np.uint8([[100, 50, 25]]), 16, 0))
    assert not out[9].any() and not out[12].any()


def test_round_cap_half_a_pixel_past_the_end():
    out = _one([10.0, 5.0, 10.0, 20.5])
    np.testing.assert_array_equal(out[10, 21], [100, 50, 25])    # d = 0.5 past the end: a = 0.5
    np.testing.assert_array_equal(out[10, 20], [200, 100, 50])


def test_zero_length_segment_is_a_disc():
    out = _one([20.0, 20.0, 20.0, 20.0], lw=4.0)              # h = 2.5
    y, x = np.mgrid[0:32, 0:40]
    d = np.sqrt(((y - 20) ** 2 + (x - 20) ** 2).astype(F))
    a = np.clip(F(2.5) - d, 0, 1)
    np.testing.assert_array_equal(out[..., 0], np.rint(a * F(200)).astype(np.uint8))
    np.testing.assert_array_equal(out[20, 22], [100, 50, 25])   # d = 2
    assert (out[20, 23] == 0).all() and (out[20, 17] == 0).all()
    np.testing.assert_array_equal(out[20, 18:23, 0], out[18:23, 20, 0])


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
@pytest.mark.parametrize("slot", [0, 1, 2, 3])
def test_non_finite_end_point_draws_nothing(bad, slot):
    seg = [10.0, 5.0, 12.0, 20.0]
    seg[slot] = bad
    np.testing.assert_array_equal(_one(seg, lw=3.0), _blank()[0])


@pytest.mark.parametrize("seg", [[-5.0, 0.0, -5.0, 39.0], [40.0, 0.0, 37.0, 39.0], [0.0, 42.5, 31.0, 42.5], [-1e30, -1e30, -1e30, 1e30]])
def test_segments_off_the_image_draw_nothing(seg):
    np.testing.assert_array_equal(_one(seg, lw=3.0), _blank()[0])


def test_later_segment_covers_an_earlier_one():
    cols = np.float32([[200.0, 0.0, 0.0], [0.0, 0.0, 255.0]])
    out = _one([[10.0, 0.0, 10.0, 39.0], [0.0, 20.0, 31.0, 20.0]], colors=cols)
    np.testing.assert_array_equal(out[10, 20], [0, 0, 255])
    np.testing.assert_array_equal(out[10, 19], [200, 0, 0])
    swapped = _one([[0.0, 20.0, 31.0, 20.0], [10.0, 0.0, 10.0, 39.0]], colors=cols[::-1].copy())
    np.testing.assert_array_equal(swapped[10, 20], [200, 0, 0])


def test_invalid_image_is_untouched():
    imgs = np.stack([_blank(v=7)[0], _blank(v=9)[0]])
    seg = np.float32([[[10.0, 5.0, 10.0, 20.0]], [[10.0, 5.0, 10.0, 20.0]]])
    out = O.draw(imgs, seg, C, 2.0, valid=np.int32([0, 1]))
    np.testing.assert_array_equal(out[0], imgs[0])
    assert (out[1] != imgs[1]).any()


def test_palette_halves_are_rounded_only_at_the_end():
    for val in (84.5, 248.5):
        k, c = np.argwhere(D.PALETTE == F(val))[0]
        cols = np.repeat(D.PALETTE[k:k + 1], 1, 0)
        full = _one([10.0, 5.0, 10.0, 20.0], colors=cols)
        assert full[10, 10, c] == np.rint(F(val)) == np.floor(val)            # rint(84.5) = 84, not the 85 a byte palette holds
        half = _one([10.5, 5.0, 10.5, 20.0], colors=cols, img=_blank(v=1))   # a = 0.5 over 1: 1 + 0.5 * (val - 1)
        assert half[10, 10, c] == np.rint(F(1) + F(0.5) * (F(val) - F(1)))


def test_background_keeps_its_bytes():
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, (1, 32, 40, 3), dtype=np.uint8)
    out = O.draw(img, np.float32([[[10.0, 5.0, 12.0, 20.0]]]), C, 2.0)[0]
    d = np.abs(np.mgrid[0:32, 0:40][0] - 11.0)
    far = d > 3
    np.testing.assert_array_equal(out[far], img[0][far])


@pytest.mark.parametrize("seed", range(4))
def test_windows_equal_the_whole_image(seed):
    """Each segment evaluated on its h + 1 box equals the rule evaluated on every pixel."""
    rng = np.random.default_rng(seed)
    imgs = rng.integers(0, 256, (2, 48, 64, 3), dtype=np.uint8)
    seg = rng.uniform(-20, 80, (2, 12, 4)).astype(F)
    seg[0, 3, 1] = np.nan
    seg[1, 5] = seg[1, 5, [0, 1, 0, 1]]                      # a point
    cols = rng.uniform(0, 255, (12, 3)).astype(F)
    for lw in (0.5, 1.0, 4.5, 13.0):
        np.testing.assert_array_equal(O.draw(imgs, seg, cols, lw), O.draw(imgs, seg, cols, lw, full=True))


@pytest.mark.parametrize("seed", range(3))
def test_windows_equal_the_whole_image_for_far_end_points(seed):
    """End points up to 2^14 px away: the box still changes nothing."""
    rng = np.random.default_rng(100 + seed)
    imgs = rng.integers(0, 256, (1, 48, 64, 3), dtype=np.uint8)
    inside = rng.uniform(0, 48, (1, 10, 2)).astype(F)
    far = rng.uniform(-16384, 16384, (1, 10, 2)).astype(F)
    seg = np.concatenate([inside, far], -1)
    cols = rng.uniform(0, 255, (10, 3)).astype(F)
    for lw in (1.0, 4.5):
        np.testing.assert_array_equal(O.draw(imgs, seg, cols, lw), O.draw(imgs, seg, cols, lw, full=True))


def test_box_is_part_of_the_rule_for_huge_end_points():
    """(10, -1e8, 10, 101) at width 1: x - c0 and c1 - c0 round to the same multiple of 8, so the box-free formula covers pixels
    (10, 104..107) past the end; the rule's box (up to column 101 + g = 103) leaves them alone."""
    seg = [10.0, -1e8, 10.0, 101.0]
    img = np.zeros((1, 20, 120, 3), np.uint8)
    boxed = _one(seg, img=img)
    free = O.draw(img, np.float32(seg).reshape(1, 1, 4), C, 1.0, full=True)[0]
    assert (free[10, 104:108] != 0).all()
    assert not boxed[10, 104:].any()                           # nothing past the box
    np.testing.assert_array_equal(boxed[10, :104], free[10, :104])


def test_projection_and_crop_box():
    xyz = np.float32([[[-3.0, -3.0, 0.0]] * 21, [[3.0, 1.0, 5.0]] * 21])
    hw = O.project_3d(xyz, 240, 360)
    np.testing.assert_array_equal(hw[0, 0], [-0.5, -0.5])
    np.testing.assert_array_equal(hw[1, 0], [239.5, 359.5])
    box = O.crop_box(np.float32([[120.0, 160.0]]), np.float32([[2.0]]))
    np.testing.assert_array_equal(box[0], [[56, 96, 56, 224], [56, 224, 184, 224], [184, 224, 184, 96], [184, 96, 56, 96]])

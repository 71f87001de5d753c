"""The numpy restatement of run.py's resize (tests/frames_oracle.py) against Pillow and against the committed golden; run.py's
normalisation over all 256 codes; the frame-coordinate mapping.  No GPU needed."""
import os

import numpy as np
import pytest

import frames_oracle as F

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_frames_pil.npz")

FRAME_SIZES = [(480, 640), (720, 1280), (1080, 1920), (2160, 3840), (241, 321), (100, 77), (3, 5), (240, 320), (1, 1), (2, 700)]
OUT_SIZES = [(240, 320), (256, 256), (320, 320)]
# integer and non-integer factors both ways, 1-pixel and prime sizes
EXTRA = [((64, 96), (32, 48)), ((64, 96), (16, 24)), ((60, 90), (7, 11)), ((7, 13), (3, 5)), ((3, 5), (7, 13)), ((13, 17), (1, 1)),
         ((1, 1), (1, 1)), ((1, 31), (5, 1)), ((97, 89), (194, 178)), ((97, 89), (101, 83)), ((31, 1), (29, 3)), ((4096, 3), (1, 2))]


def _pil(img, h, w):
    Image = pytest.importorskip("PIL.Image")
    return np.asarray(Image.fromarray(img).resize((w, h), Image.BILINEAR))


@pytest.mark.parametrize("frame_hw", FRAME_SIZES, ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("out_hw", OUT_SIZES, ids=lambda s: "to%dx%d" % s)
def test_restatement_equals_pillow(frame_hw, out_hw):
    img = np.random.default_rng(frame_hw[0] * 7919 + frame_hw[1]).integers(0, 256, frame_hw + (3,), dtype=np.uint8)
    np.testing.assert_array_equal(F.imresize(img, *out_hw), _pil(img, *out_hw))


@pytest.mark.parametrize("frame_hw,out_hw", EXTRA, ids=lambda s: "%dx%d" % s)
def test_restatement_equals_pillow_odd_factors(frame_hw, out_hw):
    img = np.random.default_rng(3).integers(0, 256, frame_hw + (3,), dtype=np.uint8)
    np.testing.assert_array_equal(F.imresize(img, *out_hw), _pil(img, *out_hw))


def test_restatement_equals_golden():
    z = np.load(GOLDEN)
    assert str(z["pillow_version"])
    for i, (H, W, h, w) in enumerate(z["cases"]):
        F.assert_equals_golden(F.imresize(F.frame(7000 + i, H, W), h, w), z, i)


def test_identity_is_a_copy_and_taps_sum_to_one():
    img = F.frame(1, 240, 320)
    np.testing.assert_array_equal(F.imresize(img, 240, 320), img)
    for n_in, n_out in [(1920, 320), (1080, 240), (77, 256), (3840, 256), (4096, 1)]:
        _, kk = F.coeffs(n_in, n_out)
        s = kk.sum(1)
        assert (np.abs(s - (1 << 22)) <= kk.shape[1]).all() and (kk >= 0).all()


def test_normalisation_of_all_codes():
    u = np.arange(256, dtype=np.uint8)
    want = np.array([np.float32(float(v) / 255.0 - 0.5) for v in range(256)], np.float32)   # Python floats are doubles
    np.testing.assert_array_equal(F.normalize(u), want)
    f32 = u.astype(np.float32) / np.float32(255.0) - np.float32(0.5)
    # float32 arithmetic is off by one ulp for half of the codes: the device uses a table built in double
    assert int((f32.view(np.int32) != want.view(np.int32)).sum()) == 128


def test_frame_coords_hand_computed():
    # (c + 0.5) * Hf / h - 0.5: the centre of the 240x320 image's first pixel is the centre of a 4.5 x 6 block of a 1080p frame
    got = F.frame_coords([[0.0, 0.0], [239.0, 319.0], [119.5, 159.5], [10.0, 20.0]], (1080, 1920))
    np.testing.assert_array_equal(got, [[1.75, 2.5], [1077.25, 1916.5], [539.5, 959.5], [46.75, 122.5]])
    np.testing.assert_array_equal(F.frame_coords([[5.0, 7.0]], (240, 320)), [[5.0, 7.0]])
    np.testing.assert_array_equal(F.frame_coords([[0.0, 0.0]], (480, 640)), [[0.5, 0.5]])

"""The numpy restatement of the camera-frame pixel formats (tests/frames_yuv_oracle.py) against OpenCV's cvtColor, against the
committed golden, and composed with the Pillow restatement of the resize.  No GPU needed."""
import os

import numpy as np
import pytest

import frames_oracle as F
import frames_yuv_oracle as Y
from hand3d_b200 import runtime

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_frames_yuv.npz")
SIZES = [(2, 2), (2, 4096), (4096, 2), (4, 6), (242, 322), (480, 640), (720, 1280), (1080, 1920), (2160, 3840), (6, 10), (98, 34)]


@pytest.mark.parametrize("fmt", Y.YUV_FORMATS + ("bgr",))
@pytest.mark.parametrize("hw", SIZES, ids=lambda s: "%dx%d" % s)
def test_restatement_equals_opencv(fmt, hw):
    cv2 = pytest.importorskip("cv2")
    f = Y.random_frame(hw[0] * 31 + hw[1], fmt, *hw)
    np.testing.assert_array_equal(Y.to_rgb(fmt, f), cv2.cvtColor(f, Y.cv2_code(cv2, fmt)))


def test_restatement_equals_golden():
    z = np.load(GOLDEN)
    assert str(z["opencv_version"])
    for i, (fmt, (H, W), seed) in enumerate(zip(z["formats"], z["sizes"], z["seeds"])):
        F.assert_equals_golden(Y.to_rgb(str(fmt), Y.random_frame(int(seed), str(fmt), int(H), int(W))), z, i)


@pytest.mark.parametrize("fmt", Y.YUV_FORMATS)
def test_layouts_round_trip(fmt):
    f = Y.random_frame(5, fmt, 6, 10)
    assert f.shape == runtime.frame_shape(fmt, 6, 10) == Y.frame_shape(fmt, 6, 10)
    np.testing.assert_array_equal(Y.pack(fmt, *Y.planes(fmt, f)), f)
    assert Y.picture_hw(fmt, f) == (6, 10)


def test_extreme_codes():
    # the corners of the YUV cube: clipping at both ends, Y below 16, and the largest intermediates (they must fit in int32)
    v = np.array([0, 15, 16, 17, 128, 235, 240, 255], np.uint8)
    Yv, U, V = [a.reshape(1, -1) for a in np.meshgrid(v, v, v, indexing="ij")]
    got = Y.yuv_to_rgb(Yv, U, V)
    c = np.maximum(Yv.astype(np.int64) - 16, 0) * Y.CY + (1 << 19)
    u, w = U.astype(np.int64) - 128, V.astype(np.int64) - 128
    want = np.clip(np.stack([c + Y.CRV * w, c + Y.CGV * w + Y.CGU * u, c + Y.CBU * u], -1) >> 20, 0, 255)
    np.testing.assert_array_equal(got, want)
    assert np.abs(np.stack([c + Y.CRV * w, c + Y.CGV * w + Y.CGU * u, c + Y.CBU * u])).max() < 2 ** 31


@pytest.mark.parametrize("fmt", Y.YUV_FORMATS)
@pytest.mark.parametrize("hw,out", [((242, 322), (240, 320)), ((480, 640), (240, 320)), ((66, 90), (256, 256)), ((10, 8), (3, 5))],
                         ids=lambda s: "%dx%d" % s)
def test_restatement_then_pillow(fmt, hw, out):
    Image = pytest.importorskip("PIL.Image")
    f = Y.random_frame(hw[0] + 3 * hw[1], fmt, *hw)
    rgb = Y.to_rgb(fmt, f)
    want = np.asarray(Image.fromarray(rgb).resize((out[1], out[0]), Image.BILINEAR))
    np.testing.assert_array_equal(Y.resize(fmt, f, *out), want)
    np.testing.assert_array_equal(Y.resize(fmt, f, *out), F.imresize(rgb, *out))


def test_frame_shape_refusals():
    for fmt, H, W in [("nv12", 3, 4), ("nv12", 4, 3), ("i420", 5, 6), ("yuyv", 4, 5), ("rgba", 4, 4)]:
        with pytest.raises(ValueError):
            runtime.frame_shape(fmt, H, W)
    assert runtime.frame_shape("yuyv", 3, 4) == (3, 4, 2) and runtime.frame_shape("bgr", 3, 5) == (3, 5, 3)

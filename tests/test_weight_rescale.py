"""The function-preserving rescaling of tests/weight_rescale.py, pinned on the fp64 oracle: with per-channel exponents in [-16, 16]
the four networks compute what the unscaled weights compute.  tests/test_gpu_tc_range.py relies on it for its metamorphic test, so a
failure there cannot come from the helper."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import weight_rescale as WR  # noqa: E402
from hand3d_b200 import weights as Wt  # noqa: E402
from oracle import hand3d_oracle as O  # noqa: E402

f64 = np.float64
E = 16


def _scaled():
    wd = Wt.synthetic_weights(0)
    ws, exps = WR.rescale(wd, E, seed=3)
    return wd, ws, exps


def test_rescale_touches_every_hidden_layer_and_no_score_layer():
    wd, ws, exps = _scaled()
    score = {"HandSegNet/conv6_2", "PoseNet2D/conv5_2", "PoseNet2D/conv6_7", "PoseNet2D/conv7_7", "PosePrior/fc_xyz",
             "ViewpointNet/fc_vp_ux", "ViewpointNet/fc_vp_uy", "ViewpointNet/fc_vp_uz"}
    for name in wd:
        if name.endswith("/biases"):
            layer = name[:-len("/biases")]
            assert np.array_equal(ws[name], wd[name]) == (layer not in exps), name
    for layer, e in exps.items():
        assert layer not in score
        assert e.min() < -E // 2 and e.max() > E // 2, layer        # the exponents really span the range
    assert len(exps) == 15 + 28 + 8 + 8
    # hand_side rows and the score-map channels of conv6_1 / conv7_1 carry only their own layer's output scale
    for n, rows in (("PosePrior/fc_rel0", slice(2048, None)), ("ViewpointNet/fc_vp0", slice(4096, None))):
        assert np.array_equal(ws[n + "/weights"][rows], np.ldexp(wd[n + "/weights"][rows], exps[n]))
    for u in (6, 7):
        n = "PoseNet2D/conv%d_1" % u
        assert np.array_equal(ws[n + "/weights"][:, :, :21], np.ldexp(wd[n + "/weights"][:, :, :21], exps[n]))


def _close(a, b):
    np.testing.assert_allclose(a, b, rtol=1e-12, atol=1e-12 * np.abs(b).max())


def test_rescaled_handsegnet_oracle():
    wd, ws, _ = _scaled()
    img = Wt.synthetic_images(2, 32, 40, seed=4)
    _close(O.inference_detection(img, ws, f64)[-1], O.inference_detection(img, wd, f64)[-1])


def test_rescaled_posenet_oracle():
    wd, ws, _ = _scaled()
    crop = Wt.synthetic_images(1, 32, 32, seed=5)
    for a, b in zip(O.inference_pose2d(crop, ws, f64), O.inference_pose2d(crop, wd, f64)):
        _close(a, b)


def test_rescaled_pose_prior_oracle():
    wd, ws, _ = _scaled()
    rng = np.random.default_rng(6)
    sm = rng.normal(size=(2, 256, 256, 21)).astype(np.float32)
    hs = Wt.synthetic_hand_side(2, seed=7)
    for variant in ("proposed", "direct"):
        got, want = O.pose_prior_inference(sm, hs, ws, variant, f64), O.pose_prior_inference(sm, hs, wd, variant, f64)
        for a, b in zip(got, want):
            if b is not None:
                _close(a, b)

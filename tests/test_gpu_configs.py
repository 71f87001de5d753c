"""GPU parity at the BASELINE.json configurations' own batch sizes, against the CPU oracle (never CUDA against CUDA):
config 2 (PoseNet-only, 32 crops of 256x256), config 3 (inference2d, 64 images of 320x320), config 5 (single-pass fp16 full
pipeline, 64 images, tolerance 1e-2) and the fp32-parity full pipeline over 64 images with its free-running mismatch rates.
The thresholds on the rates are rates measured with scripts/mismatch_report.py plus a small margin; the continuous tolerances
are BASELINE.json's (1e-3 fp32 parity, 1e-2 fp16)."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import parity_stats as PS  # noqa: E402
from hand3d_b200 import weights as Wt  # noqa: E402
from oracle import hand3d_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def wd():
    return Wt.synthetic_weights(0)


@pytest.fixture(scope="module")
def ctx(wd):
    from hand3d_b200 import runtime
    c = runtime.default_context()
    c.load_weights(wd)
    yield c
    c.set_precision("bf16x3")


@pytest.fixture(scope="module")
def full64(wd):
    img = PS.mixed_images(64, seed=21)
    hs = Wt.synthetic_hand_side(64, seed=22)
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    return img, hs, O.inference(img, hs, wd, literal_mask=False)


@pytest.fixture(scope="module")
def crops32(wd):
    crops = Wt.synthetic_images(32, 256, 256, seed=23)
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    return crops, PS.posenet_reference(crops, wd)


@pytest.mark.parametrize("prec,tol", [("bf16x3", 1e-3), ("fp16x3", 1e-3), ("fp16", 1e-2)])
def test_config2_posenet_only_batch32(ctx, wd, crops32, prec, tol):
    crops, ref_map = crops32
    st = PS.posenet_stats(ctx, crops, wd, ref_map, prec)
    print("config 2 / %s: %s" % (prec, st))
    assert st["max_abs_err_keypoints_scoremap"] < tol
    assert st["max_margin_of_differing_keypoints"] < 2 * tol, "a key-point index differs from the oracle's without a near-tie"
    assert st["keypoints_identical_rate"] >= (0.995 if tol == 1e-3 else 0.95)


@pytest.mark.parametrize("prec,tol", [("bf16x3", 1e-3), ("fp16x3", 1e-3), ("fp16", 1e-2)])
def test_full_pipeline_batch64_vs_oracle(ctx, wd, full64, prec, tol):
    """configs 4 / 5 at 64 images per GPU: teacher-forced continuous outputs within BASELINE.json's tolerance of the oracle,
    key-point indices identical except at near-ties of the oracle map, free-running crop-parameter agreement rate."""
    img, hs, ref = full64
    st = PS.full_pipeline_stats(ctx, img, hs, wd, ref, prec)
    print("full pipeline / %s: %s" % (prec, st))
    assert st["max_abs_err_hand_scoremap"] < tol
    assert st["max_abs_err_keypoints_scoremap"] < tol
    assert st["max_abs_err_coord3d"] < tol
    assert st["max_margin_of_differing_keypoints"] < 2 * tol
    assert st["keypoints_identical_forced_rate"] >= (0.995 if tol == 1e-3 else 0.95)
    assert st["crop_params_agree_rate"] >= (0.9 if tol == 1e-3 else 0.5)


def test_config3_inference2d_batch64(ctx, wd, full64):
    """eval2d.py:58: net.inference2d on 64 images of 320x320 against the oracle's inference2d (free-running)."""
    from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork
    img, _, ref = full64
    ctx.set_precision("bf16x3")
    net = ColorHandPose3DNetwork()
    kps, crop, scale, center = net.inference2d(PS.dev(img))
    kps, crop, scale, center = [t.cpu().numpy() for t in (kps, crop, scale, center)]
    assert kps.shape == (64, 256, 256, 21) and crop.shape == (64, 256, 256, 3)
    ok = (center == ref[3]).all(1) & (scale == ref[2]).all(1)
    print("config 3: crop parameters agree with the free-running oracle for %d/64 images" % int(ok.sum()))
    assert ok.mean() >= 0.9
    np.testing.assert_array_equal(crop[ok], ref[1][ok])
    assert np.abs(kps[ok] - ref[4][ok]).max() < 1e-3
    same, tot, margins = PS.keypoint_stats(net.last_keypoints_uv.cpu().numpy()[ok], kps[ok], ref[4][ok])
    assert same >= 0.995 * tot and (not margins or max(margins) < 2e-3)

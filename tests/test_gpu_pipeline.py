"""GPU parity of the network stages and of the full pipeline against the CPU oracle (reference API level).

Tolerances follow BASELINE.json: key-point indices bit-exact, fp32 score maps / 3-D coordinates within
1e-3 abs for the fp32-parity modes (fp32_ffma, bf16x3, fp16x3) and 1e-2 for the single-pass fp16 mode."""
import numpy as np
import pytest
import torch

from hand3d_b200 import weights as Wt
from oracle import hand3d_oracle as O
from oracle import tf1_ops as T

pytestmark = pytest.mark.gpu
f32 = np.float32
PARITY_MODES = ["fp32_ffma", "bf16x3", "fp16x3", "fp16_f8c"]
TOL = {"fp32_ffma": 1e-3, "bf16x3": 1e-3, "fp16x3": 1e-3, "fp16_f8c": 1e-3, "fp16": 1e-2}


@pytest.fixture(scope="module")
def wd():
    return Wt.synthetic_weights(0)


@pytest.fixture(scope="module")
def net(wd):
    from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork
    n = ColorHandPose3DNetwork()
    n.init(None, weights=wd)
    return n


@pytest.fixture(scope="module")
def ctx(net):
    from hand3d_b200 import runtime
    return runtime.default_context()


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope="module")
def seg_ref(wd):
    img = np.concatenate([Wt.synthetic_images(1, 320, 320, seed=1), Wt.synthetic_blob_images(1, 320, 320, seed=5)], 0)
    return img, O.inference_detection(img, wd)[-1]


@pytest.mark.parametrize("prec", PARITY_MODES + ["fp16"])
def test_handsegnet_stage(net, ctx, seg_ref, prec):
    img, ref = seg_ref
    ctx.set_precision(prec)
    out = net.inference_detection(_dev(img))
    assert isinstance(out, list) and len(out) == 1 and tuple(out[0].shape) == (2, 320, 320, 2)
    err = np.abs(out[0].cpu().numpy() - ref).max()
    assert err < TOL[prec], "HandSegNet %s: max abs err %.3e" % (prec, err)


def test_first_layer_ffma_kernel(net, ctx, seg_ref):
    """conv1_1 as the register-tiled FFMA kernel (c3_ffma = 1) instead of the tensor cores (conv_c3_tc_kernel, the default that
    test_handsegnet_stage runs) must give the HandSegNet parity too."""
    img, ref = seg_ref
    ctx.set_precision("bf16x3")
    ctx.set_tuning("c3_ffma", 1)
    try:
        out = net.inference_detection(_dev(img))[0].cpu().numpy()
    finally:
        ctx.set_tuning("c3_ffma", 0)
    assert np.abs(out - ref).max() < 1e-3


@pytest.mark.parametrize("prec", ["bf16x3", "fp16x3"])
@pytest.mark.parametrize("shape", [(3, 40, 40), (1, 24, 56), (2, 72, 48)])
def test_handsegnet_small_odd_maps(net, ctx, wd, shape, prec):
    """Maps that are no multiple of the pixel tile, odd numbers of tiles and tiles that lie entirely in conv1_2's zero padding:
    exercises the masking of the first-layer and the implicit-GEMM kernels."""
    B, H, W = shape
    img = Wt.synthetic_images(B, H, W, seed=17)
    ctx.set_precision(prec)
    out = net.inference_detection(_dev(img))[0].cpu().numpy()
    ref = O.inference_detection(img, wd)[-1]
    assert out.shape == (B, H, W, 2)
    assert np.abs(out - ref).max() < 1e-3


def test_handsegnet_240x320(net, ctx, wd):
    img = Wt.synthetic_images(1, 240, 320, seed=7)
    ctx.set_precision("bf16x3")
    out = net.inference_detection(_dev(img))[0].cpu().numpy()
    ref = O.inference_detection(img, wd)[-1]
    assert out.shape == (1, 240, 320, 2)
    assert np.abs(out - ref).max() < 1e-3


@pytest.fixture(scope="module")
def pose_ref(wd):
    crop = Wt.synthetic_images(2, 256, 256, seed=11)
    return crop, O.inference_pose2d(crop, wd)


@pytest.mark.parametrize("prec", PARITY_MODES + ["fp16"])
def test_posenet_stage(net, ctx, pose_ref, prec):
    crop, ref = pose_ref
    ctx.set_precision(prec)
    outs = net.inference_pose2d(_dev(crop))
    assert len(outs) == 3
    for i in range(3):
        err = np.abs(outs[i].cpu().numpy() - ref[i]).max()
        assert err < TOL[prec], "PoseNet %s stage %d: max abs err %.3e" % (prec, i, err)


# fp32_ffma: fp32 CUDA-core pyramids; bf16x3 / fp16x3: wgmma pyramids (stride 2 = odd pixels of the stride-1 result), branches on two streams
@pytest.mark.parametrize("prec", ["fp32_ffma", "bf16x3", "fp16x3"])
@pytest.mark.parametrize("variant", ["proposed", "direct"])
def test_lifting_stage(ctx, wd, variant, prec):
    rng = np.random.default_rng(13)
    B = 5
    sm = rng.normal(size=(B, 32, 32, 21)).astype(f32)
    hs = Wt.synthetic_hand_side(B, seed=3)
    ctx.set_precision(prec)
    try:
        out, can, rot = ctx.lifting(_dev(sm), _dev(hs), variant)
        out2, can2, rot2 = ctx.lifting(_dev(sm), _dev(hs), variant)     # second call: same plan, same streams
    finally:
        ctx.set_precision("bf16x3")
    tol = 1e-4 if prec == "fp32_ffma" else 3e-4
    if variant == "proposed":
        r_out, r_can, r_R = O.inference_pose3d(sm, hs, wd)
        np.testing.assert_allclose(rot.cpu().numpy(), r_R, atol=tol)
    else:
        r_can = O.inference_pose3d_can(sm, hs, wd)
        r_out = r_can
    np.testing.assert_allclose(can.cpu().numpy(), r_can, atol=tol)
    np.testing.assert_allclose(out.cpu().numpy(), r_out, atol=tol)
    assert torch.equal(out, out2) and torch.equal(can, can2)            # deterministic across calls (no atomics, no stream races)


def test_pose_prior_network_variants(wd):
    from hand3d_b200 import runtime
    from hand3d_b200.nets.PosePriorNetwork import PosePriorNetwork
    rng = np.random.default_rng(14)
    B = 3
    sm = rng.normal(size=(B, 256, 256, 21)).astype(f32)
    hs = Wt.synthetic_hand_side(B, seed=4)
    for variant in ("proposed", "direct"):
        p = PosePriorNetwork(variant)
        p.init(None, weights={k: v for k, v in wd.items() if k.startswith(("PosePrior", "ViewpointNet"))})
        out, c3, R = p.inference(_dev(sm), _dev(hs), True)
        ref = O.pose_prior_inference(sm, hs, wd, variant)
        np.testing.assert_allclose(out.cpu().numpy(), ref[0], atol=1e-4)
        np.testing.assert_allclose(c3.cpu().numpy(), ref[1], atol=1e-4)
        assert (R is None) == (ref[2] is None)
    wb = Wt.synthetic_weights(0, bottleneck=True)
    p = PosePriorNetwork("bottleneck")
    p.init(None, weights={k: v for k, v in wb.items() if k.startswith("PosePrior")})
    out, _, _ = p.inference(_dev(sm), _dev(hs), True)
    np.testing.assert_allclose(out.cpu().numpy(), O.pose_prior_inference(sm, hs, wb, "bottleneck")[0], atol=1e-4)
    # restore the standard weights for the tests that follow
    runtime.default_context().load_weights({k: v for k, v in wd.items() if k.startswith("PosePrior")})
    for variant in ("local", "local_w_xyz_loss"):      # bone_rel_trafo_inv on device (utils/relative_trafo.py:243-295)
        p = PosePriorNetwork(variant)
        out, c3, R = p.inference(_dev(sm), _dev(hs), True)
        ref = O.pose_prior_inference(sm, hs, wd, variant)
        np.testing.assert_allclose(c3.cpu().numpy(), ref[1], atol=1e-4)
        np.testing.assert_allclose(out.cpu().numpy(), ref[0], atol=1e-3)
        assert R is None
    with pytest.raises(AssertionError):
        PosePriorNetwork("nonsense").inference(_dev(sm), _dev(hs), True)


def _pipeline_case(kind):
    if kind == "noise":
        return Wt.synthetic_images(3, 320, 320, seed=1), Wt.synthetic_weights(0)
    return Wt.synthetic_blob_images(3, 320, 320, seed=5), Wt.synthetic_weights(0, seg_shift=0.15)


@pytest.mark.parametrize("kind", ["noise", "blobs"])
@pytest.mark.parametrize("prec", PARITY_MODES)
def test_full_pipeline(kind, prec):
    """inference(): stage-wise parity with the oracle.

    Continuous outputs must be within 1e-3 of the oracle; every discrete stage (mask growing, bounding box, crop
    parameters, crop, arg-max) must be EXACTLY what the oracle computes from the same inputs.  The free-running
    end-to-end agreement of the crop parameters is reported as a rate: one mask pixel whose logit gap is below the
    numerical noise may legitimately flip (SURVEY.md section 7, "discrete decisions amplify 1e-6 differences")."""
    from hand3d_b200 import runtime
    from hand3d_b200.utils.general import detect_keypoints, trafo_coords
    img, w = _pipeline_case(kind)
    B = img.shape[0]
    hs = Wt.synthetic_hand_side(B, seed=2)
    ctx = runtime.default_context()
    ctx.load_weights(w)
    ctx.set_precision(prec)
    r = ctx.pipeline(_dev(img), _dev(hs), True, want_mask=True)
    g = {k: v.cpu().numpy() for k, v in r.items() if v is not None}
    ref = O.inference(img, hs, w, literal_mask=False)
    # 1. HandSegNet logits
    assert np.abs(g["hand_scoremap"] - ref[0]).max() < 1e-3
    # 2. mask / bbox / scale: exact functions of the device's own logits
    mask_o = O.single_obj_scoremap(g["hand_scoremap"], literal=False)
    center_o, _, size_o = O.calc_center_bb(mask_o)
    np.testing.assert_array_equal(g["hand_mask"], mask_o[..., 0].astype(np.uint8))
    np.testing.assert_array_equal(g["center"], center_o)
    np.testing.assert_array_equal(g["scale_crop"], O.crop_scale(size_o))
    # 3. crop: bit-exact given the crop parameters
    np.testing.assert_array_equal(g["image_crop"], O.crop_image_from_xy(img, g["center"], 256, g["scale_crop"]))
    # 4./5. PoseNet + lifting + up-sampling against the oracle teacher-forced with the device's crop parameters
    ref_tf = O.inference(img, hs, w, literal_mask=False, forced_crop=(g["center"], g["scale_crop"]))
    np.testing.assert_array_equal(ref_tf[1], g["image_crop"])
    assert np.abs(g["keypoints_scoremap"] - ref_tf[4]).max() < 1e-3
    assert np.abs(g["keypoint_coord3d"] - ref_tf[5]).max() < 1e-3
    # 6. key-points: exact arg-max of the device map; equal to the oracle's unless the oracle map has a near-tie
    n_same = 0
    for b in range(B):
        np.testing.assert_array_equal(g["keypoints_uv"][b], O.detect_keypoints(g["keypoints_scoremap"][b]).astype(np.int32))
        np.testing.assert_array_equal(detect_keypoints(g["keypoints_scoremap"][b]), O.detect_keypoints(g["keypoints_scoremap"][b]))
        kp_ref = O.detect_keypoints(ref_tf[4][b]).astype(np.int32)
        for c in range(21):
            if np.array_equal(g["keypoints_uv"][b, c], kp_ref[c]):
                n_same += 1
            else:
                v, u = g["keypoints_uv"][b, c]
                assert ref_tf[4][b, :, :, c].max() - ref_tf[4][b, v, u, c] < 2e-3, "key-point differs without a near-tie"
        np.testing.assert_allclose(trafo_coords(detect_keypoints(g["keypoints_scoremap"][b]), g["center"][b:b + 1], g["scale_crop"][b:b + 1], 256),
                                   O.trafo_coords(O.detect_keypoints(g["keypoints_scoremap"][b]), g["center"][b:b + 1], g["scale_crop"][b:b + 1], 256))
    # 7. free-running agreement with the oracle's own discrete decisions
    agree = (g["center"] == ref[3]).all(1) & (g["scale_crop"] == ref[2]).all(1)
    print("%s/%s: crop parameters agree with the free-running oracle for %d/%d images; key-points identical %d/%d"
          % (kind, prec, int(agree.sum()), B, n_same, 21 * B))
    assert agree.mean() >= 0.5
    assert n_same >= 21 * B - 2
    if kind == "blobs":
        assert len(np.unique(g["scale_crop"])) > 1, "the blob set is meant to give varied crops"


def test_reference_api_tuple_orders(wd):
    from hand3d_b200 import runtime
    from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork
    img = Wt.synthetic_images(1, 320, 320, seed=1)
    hs = Wt.synthetic_hand_side(1, seed=2)
    net = ColorHandPose3DNetwork()
    net.init(None, weights=wd)
    runtime.default_context().set_precision("bf16x3")
    out = net.inference(_dev(img), _dev(hs), torch.tensor(True))
    shapes = [tuple(o.shape) for o in out]
    assert shapes == [(1, 320, 320, 2), (1, 256, 256, 3), (1, 1), (1, 2), (1, 256, 256, 21), (1, 21, 3)]
    with pytest.raises(NotImplementedError):
        net.inference(_dev(img), _dev(hs), False)


def test_inference2d_tuple_order_and_teacher_forcing(wd):
    from hand3d_b200 import runtime
    from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork
    img = Wt.synthetic_images(2, 240, 320, seed=9)
    net = ColorHandPose3DNetwork()
    net.init(None, weights=wd, exclude_var_list=['PosePrior', 'ViewpointNet'])     # eval2d.py:78-79
    ctx = runtime.default_context()
    ctx.set_precision("bf16x3")
    kps, crop, scale, center = net.inference2d(_dev(img))
    r = O.inference2d(img, wd, literal_mask=False)
    assert tuple(kps.shape) == (2, 256, 256, 21) and tuple(crop.shape) == (2, 256, 256, 3)
    np.testing.assert_array_equal(center.cpu().numpy(), r[3])
    np.testing.assert_array_equal(scale.cpu().numpy(), r[2])
    assert np.abs(kps.cpu().numpy() - r[0]).max() < 1e-3
    # teacher-forced crop parameters
    fc = np.array([[100.0, 120.0], [200.0, 50.0]], f32); fs = np.array([[1.5], [0.7]], f32)
    hs = Wt.synthetic_hand_side(2, seed=1)
    res = ctx.pipeline(_dev(img), _dev(hs), True, force_center=_dev(fc), force_scale=_dev(fs))
    ref = O.inference(img, hs, wd, forced_crop=(fc, fs))
    np.testing.assert_array_equal(res["image_crop"].cpu().numpy(), ref[1])
    assert np.abs(res["keypoint_coord3d"].cpu().numpy() - ref[5]).max() < 1e-3


def test_unknown_variable_and_bad_numerics(ctx):
    with pytest.raises(ValueError):
        ctx.load_weights({"HandSegNet/conv9_9/weights": np.zeros((3, 3, 3, 3), f32)})
    with pytest.raises(ValueError):
        ctx.load_weights({"HandSegNet/conv1_1/weights": np.zeros((3, 3, 4, 64), f32)})
    bad = np.zeros((512, 63), f32); bad[0, 0] = np.nan
    with pytest.raises(ValueError):
        ctx.load_weights({"PosePrior/fc_xyz/weights": bad})


def test_example_drivers_run():
    """The run.py / eval2d.py shaped drivers (examples/) execute end to end on synthetic data."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for script, args in (("run_demo.py", []), ("eval2d_demo.py", ["--samples", "8", "--batch", "4"]),
                         ("eval2d_gt_cropped_demo.py", ["--samples", "8", "--batch", "4"]), ("eval3d_demo.py", ["--samples", "8", "--batch", "4"]),
                         ("eval3d_demo.py", ["--samples", "4", "--batch", "4", "--variant", "proposed"]),
                         ("eval_full_demo.py", ["--samples", "4", "--batch", "2"])):
        r = subprocess.run([sys.executable, os.path.join(root, "examples", script)] + args, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, (script, r.stderr[-2000:])
        assert ("3D wrist" in r.stdout) or ("Area under curve" in r.stdout), r.stdout

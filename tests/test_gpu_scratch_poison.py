"""No result may depend on memory the call did not write: every entry point run on a poisoned workspace and operator scratch.

The stage workspace (h3d_set_workspace) and the context's operator scratch carry no state between calls (include/hand3d_b200.h).
Several results are only right because a region holds zeros or finite values before the call: the K padding channels the
tensor-core layers read (PoseNet2D's concat channels 149..191, the lifting pyramids' 21 -> 64 and 32 -> 64 channels, the FC stacks'
padded columns) meet zero weights, so a finite stale value there vanishes and fresh cudaMalloc pages are zero anyway.  Only a
non-finite value makes a lost write visible, and the max-pools' fmaxf drops NaN.  So every scenario runs three times, after
h3d_fill_scratch with
  0x00  zeros;
  0xFF  NaN in fp32, bf16, fp16 and e4m3;
  0x7B  finite and huge in every format (1.3e36 in fp32 and bf16, 61280 in fp16, 352 in e4m3), which no fmaxf can drop,
and all outputs must be bit-identical.  As a second line of defence the poisoned outputs are also held against the oracle or the
fp64 references at the tolerances of the existing tests.  The scratch grows on demand, so each scenario is run once before the
three filled runs.

The 95 cases take 56 s on one NVIDIA H100 80GB HBM3 (power limit 700 W).

Two deliberately wrong builds survive this module, and test_gpu_pipeline.py and test_gpu_lifting.py too, because each removes one
of two writes of the same zeros: without the per-call memset of PoseNet2D's concat buffer, the conv5_2 head's epilogue still writes
all 64 plane channels 128..191, zeros at 149..191; without that epilogue's explicit zeroing, the padding output channels still get
the accumulator plus bias of all-zero weight rows and a zero bias, an exact zero for finite inputs.  Either alone is redundant;
removing a write that nothing else makes (a region read but never written) is what the fills expose."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

import train_oracle as TO
from hand3d_b200 import weights as Wt
from oracle import hand3d_oracle as O
from oracle import tf1_grads as G
from oracle import tf1_ops as T

pytestmark = pytest.mark.gpu
f32, f64 = np.float32, np.float64

PATTERNS = (0x00, 0xFF, 0x7B)
PRECISIONS = ["fp32_ffma", "bf16x3", "fp16x3", "fp16", "bf16", "fp16_f8c"]
# pipeline outputs against the oracle (test_gpu_pipeline.py, test_gpu_configs.py); the suite pins no pipeline-level bound for bf16,
# so there only the exact checks against the device's own intermediate values apply
PIPE_TOL = {"fp32_ffma": 1e-3, "bf16x3": 1e-3, "fp16x3": 1e-3, "fp16_f8c": 1e-3, "fp16": 1e-2}
# tensor-core operators on outputs of unit scale (test_gpu_tc_conv.py) and their gradients (test_gpu_conv_backward.py)
TC_TOL = {"bf16x3": 5e-5, "fp16x3": 2e-5, "fp16": 6e-3, "bf16": 5e-2, "fp16_f8c": 2e-4}
BWD_TOL = {"bf16x3": {"dx": 5e-5, "dw": 1e-4, "db": 1e-4}, "bf16": {"dx": 5e-2, "dw": 5e-2, "db": 5e-2}}
# lifting, normwise per output (test_gpu_lifting.py): the wgmma paths and the fp32 CUDA-core path
LIFT_BOUND = {"tc": {"out": 1.8e-4, "can": 8.2e-5, "rot": 1.9e-4}, "ffma": {"out": 1.2e-5, "can": 4.1e-6, "rot": 1.5e-5}}
# lifting kernel paths: precision, tuning switches, bound
LIFT_PATHS = {
    "tensor": ("bf16x3", {}, "tc"),
    "fc_chain0": ("bf16x3", {"fc_chain": 0}, "tc"),
    "lift_direct": ("bf16x3", {"lift_direct": 1}, "ffma"),
    "fp32_ffma": ("fp32_ffma", {}, "ffma"),
}
TUNING_DEFAULTS = {"fc_chain": 1, "lift_direct": 0}
# canaries of the output test: NaN payloads in fp32, an impossible key-point index, an impossible mask byte
CANARY32, CANARY_UV, CANARY8 = 0x7FC0A5A5, -0x5A5A5A5B, 0xA5

WD = Wt.synthetic_weights(0, seg_shift=0.15)
W_LIFT = {k: v for k, v in Wt.synthetic_weights(0).items() if k.startswith(("PosePrior", "ViewpointNet"))}
W_BOTT = {k: v for k, v in Wt.synthetic_weights(0, bottleneck=True).items() if k.startswith("PosePrior")}


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _snap(r):
    """Clones the tensors of a result (dict, tuple or tensor) into a flat dict."""
    if isinstance(r, torch.Tensor):
        r = {"out": r}
    elif isinstance(r, (list, tuple)):
        r = {str(i): t for i, t in enumerate(r)}
    return {k: t.detach().clone() for k, t in r.items() if isinstance(t, torch.Tensor)}


def _bits(t):
    return t.detach().contiguous().reshape(-1).view(torch.uint8)


def _assert_same_bits(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, what
    if not torch.equal(_bits(a), _bits(b)):
        diff = (_bits(a) != _bits(b)).nonzero()
        raise AssertionError("%s differs in %d bytes (first at byte %d)" % (what, diff.numel(), int(diff[0])))


def _poisoned_runs(ctx, fn):
    """fn() once to size the scratch, build the plans and pack the weights, then once after each fill of PATTERNS: returns the
    three snapshots, asserted bit-identical."""
    fn()
    torch.cuda.synchronize()
    runs = []
    for byte in PATTERNS:
        ctx.fill_scratch(byte)
        runs.append(_snap(fn()))
    torch.cuda.synchronize()
    ctx.check_errors()
    for byte, r in zip(PATTERNS[1:], runs[1:]):
        assert set(r) == set(runs[0])
        for k in runs[0]:
            _assert_same_bits(r[k], runs[0][k], "%s after filling the scratch with 0x%02X" % (k, byte))
    return runs


def _err(g, ref):
    return float(np.abs(np.asarray(g, f64) - ref).max() / max(np.abs(ref).max(), 1e-30))


def _new_context(weights, precision="bf16x3"):
    from hand3d_b200 import runtime
    c = runtime.Context()
    c.load_weights(weights)
    c.set_precision(precision)
    return c


def _destroy(c):
    torch.cuda.synchronize()
    c.lib.h3d_destroy(c.h)
    c.h = None
    c._ws = None


@pytest.fixture(scope="module")
def ctx():
    """A fresh process-wide default context (the network classes and the train=True graphs use that one), restored afterwards."""
    from hand3d_b200 import runtime
    from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork
    saved = dict(runtime._default)
    runtime._default.clear()
    ColorHandPose3DNetwork().init(None, weights=WD)
    c = runtime.default_context()
    c.set_precision("bf16x3")
    yield c
    torch.cuda.synchronize()
    for k, v in TUNING_DEFAULTS.items():
        c.set_tuning(k, v)
    _destroy(c)
    runtime._default.clear()
    runtime._default.update(saved)
    gc.collect()
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------- pipeline
def _check_pipeline_vs_oracle(g, img, hs, prec, forced=None):
    """The second line of defence, as test_full_pipeline: HandSegNet's logits against the oracle; mask, box, scale, crop and
    key-points exactly what the oracle computes from the device's own values; PoseNet2D, the up-sampling and the lifting against
    the oracle teacher-forced with the device's crop."""
    g = {k: v.cpu().numpy() for k, v in g.items()}
    tol = PIPE_TOL.get(prec)
    if forced is None:
        if tol is not None:
            assert np.abs(g["hand_scoremap"] - O.inference_detection(img, WD)[-1]).max() < tol
        mask_o = O.single_obj_scoremap(g["hand_scoremap"], literal=False)
        center_o, _, size_o = O.calc_center_bb(mask_o)
        np.testing.assert_array_equal(g["hand_mask"], mask_o[..., 0].astype(np.uint8))
        np.testing.assert_array_equal(g["center"], center_o)
        np.testing.assert_array_equal(g["scale_crop"], O.crop_scale(size_o))
    else:
        np.testing.assert_array_equal(g["center"], forced[0])
        np.testing.assert_array_equal(g["scale_crop"], forced[1])
    np.testing.assert_array_equal(g["image_crop"], O.crop_image_from_xy(img, g["center"], 256, g["scale_crop"]))
    for b in range(img.shape[0]):
        np.testing.assert_array_equal(g["keypoints_uv"][b], O.detect_keypoints(g["keypoints_scoremap"][b]).astype(np.int32))
    if tol is not None:
        ref = O.inference(img, hs, WD, literal_mask=False, forced_crop=(g["center"], g["scale_crop"]))
        assert np.abs(g["keypoints_scoremap"] - ref[4]).max() < tol
        assert np.abs(g["keypoint_coord3d"] - ref[5]).max() < tol


def _pipeline_case(ctx, prec, img, hs, forced=None):
    ctx.set_precision(prec)
    im, h = _cu(img), _cu(hs)
    fc, fs = (None, None) if forced is None else (_cu(forced[0]), _cu(forced[1]))
    runs = _poisoned_runs(ctx, lambda: ctx.pipeline(im, h, True, force_center=fc, force_scale=fs, want_mask=True))
    assert set(runs[0]) == {"hand_scoremap", "image_crop", "scale_crop", "center", "keypoints_scoremap", "keypoint_coord3d",
                            "keypoints_uv", "hand_mask"}
    _check_pipeline_vs_oracle(runs[2], img, hs, prec, forced)


IMG_320 = Wt.synthetic_blob_images(2, 320, 320, seed=5)
IMG_240 = Wt.synthetic_blob_images(3, 240, 320, seed=6)


@pytest.mark.parametrize("prec", PRECISIONS)
def test_pipeline_b2_320x320(ctx, prec):
    _pipeline_case(ctx, prec, IMG_320, Wt.synthetic_hand_side(2, seed=2))


@pytest.mark.parametrize("prec", ["bf16x3", "fp16_f8c"])
def test_pipeline_b3_240x320(ctx, prec):
    _pipeline_case(ctx, prec, IMG_240, Wt.synthetic_hand_side(3, seed=3))


def test_pipeline_cluster_grower_600x800(ctx):
    """max(H, W) > 512: the mask grows on a thread-block cluster (mask_grow_cluster_kernel) over the seg scratch."""
    _pipeline_case(ctx, "bf16x3", Wt.synthetic_blob_images(1, 600, 800, seed=8), Wt.synthetic_hand_side(1, seed=4))


def test_pipeline_teacher_forced(ctx):
    forced = (np.array([[100.0, 120.0], [200.0, 50.0]], f32), np.array([[1.5], [0.7]], f32))
    _pipeline_case(ctx, "bf16x3", IMG_240[:2], Wt.synthetic_hand_side(2, seed=1), forced)


# ---------------------------------------------------------------------------------------------------------------- layout reuse
def test_smaller_batch_inside_a_larger_layout():
    """A plan rebuilt for B = 3 at 240x320 inside the layout of B = 8 at 480x640 reads nothing of the previous call's rows: after
    a poison between the two calls it equals a fresh context's B = 3 result bit for bit.  The same for a stand-alone PoseNet2D on
    128x128 crops after a 320x320 pipeline."""
    big = _cu(Wt.synthetic_blob_images(8, 480, 640, seed=9))
    big_hs = _cu(Wt.synthetic_hand_side(8, seed=9))
    small, small_hs = _cu(IMG_240), _cu(Wt.synthetic_hand_side(3, seed=3))
    p320, p320_hs = _cu(IMG_320), _cu(Wt.synthetic_hand_side(2, seed=2))
    crops = _cu(Wt.synthetic_images(2, 128, 128, seed=12))
    fresh = _new_context(WD)
    try:
        want = _snap(fresh.pipeline(small, small_hs, True, want_mask=True))
        want_pose = _snap(fresh.posenet(crops))
    finally:
        _destroy(fresh)
    for big_call, small_call, ref, what in (
            (lambda c: c.pipeline(big, big_hs, True, want_mask=True), lambda c: c.pipeline(small, small_hs, True, want_mask=True), want,
             "B=3 240x320 pipeline after B=8 480x640,"),
            (lambda c: c.pipeline(p320, p320_hs, True), lambda c: c.posenet(crops), want_pose,
             "PoseNet2D on 128x128 crops after a 320x320 pipeline,")):
        c = _new_context(WD)
        try:
            for byte in PATTERNS[1:]:
                big_call(c)
                c.fill_scratch(byte)
                got = _snap(small_call(c))
                for k in ref:
                    _assert_same_bits(got[k], ref[k], "%s %s after a 0x%02X fill" % (what, k, byte))
            torch.cuda.synchronize()
            c.check_errors()
        finally:
            _destroy(c)
    gc.collect()
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------- lifting
LIFT_BATCHES = [1, 13, 129]


def _lift_inputs():
    rng = np.random.default_rng(2027)
    B = max(LIFT_BATCHES)
    sm = rng.normal(size=(B, 32, 32, 21)).astype(f32)
    hs = np.zeros((B, 2), f32)
    hs[np.arange(B), rng.integers(0, 2, size=B)] = 1.0
    return sm, hs


LIFT_SM, LIFT_HS = _lift_inputs()
_LIFT_ORACLE = {}


def _lift_oracle(variant):
    if variant not in _LIFT_ORACLE:
        if variant == "proposed":
            r = O.inference_pose3d(LIFT_SM, LIFT_HS, W_LIFT, dtype=f64)
        elif variant == "bottleneck":
            c = O.inference_pose3d_can(LIFT_SM, LIFT_HS, W_BOTT, dtype=f64, bottleneck=True)
            r = (c, c, None)
        else:
            c = O.inference_pose3d_can(LIFT_SM, LIFT_HS, W_LIFT, dtype=f64)
            r = (O.bone_rel_trafo_inv(c) if variant == "local" else c, c, None)
        _LIFT_ORACLE[variant] = r
    return _LIFT_ORACLE[variant]


@pytest.fixture(scope="module")
def lift_ctx():
    """A private context: at B = 129 the workspace (sized for 256x256 PoseNet2D crops) takes several GB."""
    c = _new_context(W_LIFT)
    c.ensure_workspace(max(LIFT_BATCHES), 8, 8)
    c.weight_set = "std"
    try:
        yield c
    finally:
        for k, v in TUNING_DEFAULTS.items():
            c.set_tuning(k, v)
        _destroy(c)
        gc.collect()
        torch.cuda.empty_cache()


@pytest.mark.parametrize("path", list(LIFT_PATHS))
@pytest.mark.parametrize("B", LIFT_BATCHES)
@pytest.mark.parametrize("variant", ["proposed", "direct", "bottleneck", "local"])
def test_lifting(lift_ctx, variant, B, path):
    c = lift_ctx
    want_set = "bott" if variant == "bottleneck" else "std"
    if c.weight_set != want_set:
        c.load_weights(W_BOTT if want_set == "bott" else {k: v for k, v in W_LIFT.items() if k.startswith("PosePrior")})
        c.weight_set = want_set
    prec, switches, bound = LIFT_PATHS[path]
    c.set_precision(prec)
    try:
        for k, v in {**TUNING_DEFAULTS, **switches}.items():
            c.set_tuning(k, v)
        sm, hs = _cu(LIFT_SM[:B]), _cu(LIFT_HS[:B])
        runs = _poisoned_runs(c, lambda: c.lifting(sm, hs, variant))
    finally:
        for k, v in TUNING_DEFAULTS.items():
            c.set_tuning(k, v)
    r_out, r_can, r_rot = _lift_oracle(variant)
    g = runs[2]
    errs = {"out": _err(g["0"].cpu().numpy(), r_out[:B]), "can": _err(g["1"].cpu().numpy(), r_can[:B])}
    if r_rot is not None:
        errs["rot"] = _err(g["2"].cpu().numpy(), r_rot[:B])
    for k, e in errs.items():
        assert e <= LIFT_BOUND[bound][k], "%s: normwise error %.2e (bound %.1e)" % (k, e, LIFT_BOUND[bound][k])


# ---------------------------------------------------------------------------------------------------------------- graphs
def test_captured_pipeline_replays_on_a_poisoned_workspace(ctx):
    ctx.set_precision("bf16x3")
    img, hs = _cu(IMG_240[:2]), _cu(Wt.synthetic_hand_side(2, seed=5))
    replay, res = ctx.capture_pipeline(img, hs)
    try:
        runs = []
        for byte in PATTERNS:
            ctx.fill_scratch(byte)
            replay()
            runs.append(_snap(res))
        ctx.fill_scratch(0xFF)
        eager = _snap(ctx.pipeline(img, hs, True, outputs="keypoints"))
        torch.cuda.synchronize()
        ctx.check_errors()
    finally:
        del replay, res
        ctx.release_graphs()
    for byte, r in zip(PATTERNS, runs):
        for k in eager:
            _assert_same_bits(r[k], eager[k], "replay of %s after a 0x%02X fill" % (k, byte))


def _frame_sequence(n, B=2, H=480, W=640):
    base = np.clip((Wt.synthetic_blob_images(B, H, W, seed=13) + 0.5) * 255.0, 0, 255).astype(np.uint8)
    return [np.ascontiguousarray(np.stack([np.roll(base[b], (3 * t, 5 * t), axis=(0, 1)) for b in range(B)])) for t in range(n)]


def test_frame_runner_tracking_on_a_poisoned_workspace(ctx):
    """FrameRunner(track=True) replays a detect and a track graph per input buffer; the workspace is poisoned before every submit.
    Each step equals the eager resize + h3d_track_step on a state of its own, with the same detect / track choice."""
    from hand3d_b200 import runtime
    from hand3d_b200.frames import FrameRunner
    ctx.set_precision("bf16x3")
    frames = [_cu(f) for f in _frame_sequence(6)]
    keys = ("keypoints_uv", "keypoint_coord3d", "center", "scale_crop", "track_score", "track_lost")
    runner = FrameRunner(ctx, 2, (480, 640), track=True, redetect_every=3)
    try:
        got, detected = [], []
        for t, f in enumerate(frames):
            ctx.fill_scratch(PATTERNS[1 + t % 2])
            r = runner.submit(f)
            detected.append(r["detected"])
            got.append(_snap({k: r[k] for k in keys}))
        torch.cuda.synchronize()
    finally:
        del runner
        ctx.release_graphs()
    assert detected[0] and detected[3] and not all(detected), detected
    state = runtime.TrackState(2, ctx.device)
    hs = torch.tensor([[1.0, 0.0], [1.0, 0.0]], device=ctx.device)
    for t, f in enumerate(frames):
        ctx.fill_scratch(0x00)
        image = ctx.resize_frames(f, 240, 320, normalize=True)
        e = ctx.track_step(image, hs, state, detected[t], margin=1.5, outputs="keypoints")
        e["track_score"], e["track_lost"] = state.score.clone(), state.lost != 0
        for k in keys:
            _assert_same_bits(got[t][k], e[k], "%s at step %d (%s)" % (k, t, "detect" if detected[t] else "track"))
    ctx.check_errors()


# ---------------------------------------------------------------------------------------------------------------- operators
CONV_SHAPES = [(2, 20, 12, 100, 72, 3, 1), (1, 12, 20, 21, 40, 3, 1), (1, 12, 20, 21, 40, 3, 2)]   # K and N padding on both sides


def _conv_problem(case, seed=31):
    B, H, W, Cin, Cout, k, s = case
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(B, H, W, Cin)).astype(f32)
    w = (rng.normal(size=(k, k, Cin, Cout)) / np.sqrt(k * k * Cin)).astype(f32)
    b = (rng.normal(size=Cout) * 0.1).astype(f32)
    return x, w, b


@pytest.mark.parametrize("case", CONV_SHAPES)
@pytest.mark.parametrize("prec", ["bf16x3", "fp16x3", "fp16", "bf16", "fp16_f8c"])
def test_conv2d_tc_packed_and_device_weights(ctx, prec, case):
    x, w, b = _conv_problem(case)
    s = case[-1]
    xg = _cu(x)
    pk = ctx.pack_conv(w, b, prec)
    ref = T.leaky_relu(T.conv2d_same(x, w, b, s, f64))
    try:
        runs = _poisoned_runs(ctx, lambda: ctx.conv2d_tc_packed(xg, pk, leaky=True, stride=s))
    finally:
        del pk
    assert np.abs(runs[2]["out"].cpu().numpy() - ref).max() < TC_TOL[prec]
    if prec != "fp16_f8c":    # h3d_conv2d_tc_dev takes no fp8-correction mode
        wg, bg = _cu(w), _cu(b)
        dev = _poisoned_runs(ctx, lambda: ctx.conv2d_tc_dev(xg, wg, bg, stride=s, leaky=True, precision=prec))
        _assert_same_bits(dev[2]["out"], runs[2]["out"], "device-weight against packed result")


BWD_SHAPES = [(2, 41, 45, 64, 64, 3, 1), (2, 32, 48, 3, 64, 3, 1), (1, 12, 20, 21, 40, 3, 2), (2, 16, 16, 64, 64, 3, 2)]


@pytest.mark.parametrize("case", BWD_SHAPES)
@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
def test_conv2d_tc_backward(ctx, prec, case):
    x, w, b = _conv_problem(case, seed=21)
    s = case[-1]
    dy = np.random.default_rng(22).normal(size=(case[0], case[1] // s, case[2] // s, case[4])).astype(f32)
    xg, wg, bg, dyg = _cu(x), _cu(w), _cu(b), _cu(dy)
    y = ctx.conv2d_tc_dev(xg, wg, bg, stride=s, leaky=True, precision=prec)
    need_dx = case[3] != 3
    runs = _poisoned_runs(ctx, lambda: ctx.conv2d_tc_backward(xg, y, dyg, wg, stride=s, leaky=True, precision=prec, need_dx=need_dx))
    rdx, rdw, rdb = G.conv_grads(x, w, b, dy, s, leaky=True, pre=y.cpu().numpy())
    g = runs[2]
    errs = {"dw": _err(g["1"].cpu().numpy(), rdw), "db": _err(g["2"].cpu().numpy(), rdb)}
    if need_dx:
        errs["dx"] = _err(g["0"].cpu().numpy(), rdx)
    else:
        assert "0" not in g
    for k, e in errs.items():
        assert e < BWD_TOL[prec][k], "%s normwise error %.3e (bound %.1e)" % (k, e, BWD_TOL[prec][k])


def test_conv2d_f32_split_k(ctx):
    x, w, b = _conv_problem((1, 8, 8, 128, 256, 3, 1))
    xg, wg, bg = _cu(x), _cu(w), _cu(b)
    runs = _poisoned_runs(ctx, lambda: ctx.conv2d(xg, wg, bg, stride=1, leaky=True))
    np.testing.assert_allclose(runs[2]["out"].cpu().numpy(), T.leaky_relu(T.conv2d_same(x, w, b, 1, f64)), atol=2e-5, rtol=1e-5)


@pytest.mark.parametrize("B,n_in,n_out", [(3, 2050, 512), (33, 512, 63), (1, 4098, 256)])
def test_fully_connected(ctx, B, n_in, n_out):
    rng = np.random.default_rng(8)
    x = rng.normal(size=(B, n_in)).astype(f32)
    w = (rng.normal(size=(n_in, n_out)) / np.sqrt(n_in)).astype(f32)
    b = rng.normal(size=n_out).astype(f32)
    xg, wg, bg = _cu(x), _cu(w), _cu(b)
    runs = _poisoned_runs(ctx, lambda: ctx.fully_connected(xg, wg, bg, leaky=True))
    ref = T.fully_connected(x, w, b, f64)
    np.testing.assert_allclose(runs[2]["out"].cpu().numpy(), np.maximum(ref, 0.01 * ref), atol=2e-5, rtol=1e-5)


@pytest.mark.parametrize("H,W", [(64, 96), (600, 520)])
def test_seg_postprocess(ctx, H, W):
    rng = np.random.default_rng(H)
    low = rng.normal(size=(3, H // 8, W // 8, 2)).astype(f32) * 3.0
    low[..., 1] -= 1.5
    sm = T.resize_bilinear_tf1(low, H, W)
    smg = _cu(sm)
    runs = _poisoned_runs(ctx, lambda: ctx.seg_postprocess(smg))
    g = {k: v.cpu().numpy() for k, v in runs[2].items()}
    fg, _ = O.seg_fg_det(sm)
    mask = O.single_obj_scoremap(sm, literal=False)
    center, _, size = O.calc_center_bb(mask)
    np.testing.assert_array_equal(g["max_loc"], O.find_max_location(fg))
    np.testing.assert_array_equal(g["hand_mask"], mask[..., 0].astype(np.uint8))
    np.testing.assert_array_equal(g["center"], center)
    np.testing.assert_array_equal(g["crop_size"], size)
    np.testing.assert_array_equal(g["scale_crop"], O.crop_scale(size))


def test_detect_and_upsample_detect_keypoints(ctx):
    rng = np.random.default_rng(17)
    sm = rng.normal(size=(3, 32, 32, 21)).astype(f32)
    smg = _cu(sm)
    det = _poisoned_runs(ctx, lambda: ctx.detect_keypoints(smg))
    up = _poisoned_runs(ctx, lambda: ctx.upsample_detect_keypoints(smg, 256, 256))
    ref_up = T.resize_bilinear_tf1(sm, 256, 256)
    np.testing.assert_array_equal(up[2]["0"].cpu().numpy(), ref_up)
    for b in range(3):
        np.testing.assert_array_equal(det[2]["out"].cpu().numpy()[b], O.detect_keypoints(sm[b]).astype(np.int32))
        np.testing.assert_array_equal(up[2]["1"].cpu().numpy()[b], O.detect_keypoints(ref_up[b]).astype(np.int32))


def test_resize_backward_and_losses(ctx):
    rng = np.random.default_rng(19)
    dy = rng.normal(size=(2, 97, 41, 21)).astype(f32)
    dyg = _cu(dy)
    r = _poisoned_runs(ctx, lambda: ctx.resize_bilinear_backward(dyg, 30, 17))
    assert _err(r[2]["out"].cpu().numpy(), TO.resize_bilinear_grad(dy, 30, 17)) <= 1e-6
    P = rng.normal(size=(3, 32, 24, 21)).astype(f32)
    Tg = rng.normal(size=(3, 32, 24, 21)).astype(f32)
    vis = (rng.uniform(size=(3, 21)) > 0.3).astype(f32)
    Pc, Tc, Vc = _cu(P), _cu(Tg), _cu(vis)
    r = _poisoned_runs(ctx, lambda: ctx.scoremap_loss(Pc, Tc, Vc))
    ref_L, ref_rms = TO.scoremap_loss(P, Tg, vis)
    assert abs(float(r[2]["0"]) - ref_L) <= 1e-5 * abs(ref_L)
    assert _err(r[2]["1"].cpu().numpy(), ref_rms) <= 1e-5
    x = rng.normal(scale=4.0, size=(3, 40, 24, 2)).astype(f32)
    hand = rng.uniform(size=(3, 40, 24)) > 0.7
    lab = np.stack([~hand, hand], -1).astype(f32)
    xc, lc = _cu(x), _cu(lab)
    r = _poisoned_runs(ctx, lambda: ctx.softmax_xent(xc, lc))
    ref = TO.softmax_xent(x, lab)
    assert abs(float(r[2]["out"]) - ref) <= 1e-5 * abs(ref)


def _grads(variables):
    return {k: p.grad.detach().clone() for k, p in variables.items()}


def _train_runs(ctx, scope, step):
    """step() builds a train=True loss on `scope`'s variables and back-propagates it; the gradients of every variable must not
    depend on the scratch."""
    v = ctx.variables(scope)

    def once():
        for p in v.values():
            p.grad = None
        step()
        return _grads(v)
    runs = _poisoned_runs(ctx, once)
    assert len(runs[0]) == len(v) and all(torch.isfinite(g).all() for g in runs[0].values())


def test_train_gradients_posenet2d_and_handsegnet_64x64(ctx):
    from hand3d_b200 import autograd as A
    from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork
    ctx.set_precision("bf16x3")
    net = ColorHandPose3DNetwork()
    rng = np.random.default_rng(18)
    img = _cu(Wt.synthetic_images(2, 64, 64, seed=18))
    target = _cu(rng.uniform(size=(2, 64, 64, 21)).astype(f32) * 0.2)
    vis = _cu((rng.uniform(size=(2, 21)) > 0.2).astype(f32))
    hand = rng.uniform(size=(2, 64, 64)) > 0.7
    labels = _cu(np.stack([~hand, hand], -1).astype(f32))

    def pose_step():
        maps = net.inference_pose2d(img, train=True)
        sum(A.scoremap_loss(A.resize_bilinear(m, 64, 64), target, vis) for m in maps).backward()

    def seg_step():
        A.softmax_xent_loss(net.inference_detection(img, train=True)[0], labels).backward()
    _train_runs(ctx, "PoseNet2D", pose_step)
    _train_runs(ctx, "HandSegNet", seg_step)


def test_train_gradients_lifting(ctx):
    from hand3d_b200 import autograd as A
    from hand3d_b200.nets.PosePriorNetwork import PosePriorNetwork
    ctx.set_precision("bf16x3")
    rng = np.random.default_rng(41)
    uv = _cu(rng.uniform(20, 236, size=(8, 21, 2)).astype(f32))
    sm = ctx.gaussian_scoremap(uv, (256, 256), 25.0)
    hs = np.zeros((8, 2), f32)
    hs[np.arange(8), rng.integers(0, 2, 8)] = 1
    hs = _cu(hs)
    xyz = _cu((rng.normal(size=(8, 21, 3)) * 0.3).astype(f32))

    def step():
        _, coord3d, _ = PosePriorNetwork("direct").inference(sm, hs, train=True)
        A.mse_loss(coord3d, xyz).backward()
    _train_runs(ctx, "PosePrior", step)


# ---------------------------------------------------------------------------------------------------------------- outputs
def _canaried(shape, dtype):
    t = torch.empty(shape, dtype=dtype, device="cuda")
    if dtype == torch.float32:
        t.view(torch.int32).fill_(CANARY32)
    elif dtype == torch.int32:
        t.fill_(CANARY_UV)
    else:
        t.fill_(CANARY8)
    return t


def _assert_overwritten(outs, ref, what):
    for k, t in outs.items():
        _assert_same_bits(t, ref[k], "%s %s (canary left or value changed)" % (what, k))


def test_c_entries_overwrite_every_output_element(ctx):
    """h3d_pipeline_forward and h3d_track_step through ctypes, on a poisoned workspace, into outputs pre-filled with canaries (as
    test_operator_entries_enqueue_only calls the entries): every element is overwritten with the value the Python wrapper returns."""
    from hand3d_b200 import _lib, runtime
    ctx.set_precision("bf16x3")
    B, H, W = 3, 240, 320
    img, hs = _cu(IMG_240), _cu(Wt.synthetic_hand_side(B, seed=3))
    p = lambda t: C.c_void_p(0 if t is None else t.data_ptr())     # noqa: E731
    st = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)     # noqa: E731
    want = _snap(ctx.pipeline(img, hs, True, want_mask=True))
    shapes = {"hand_scoremap": ((B, H, W, 2), torch.float32), "image_crop": ((B, 256, 256, 3), torch.float32),
              "scale_crop": ((B, 1), torch.float32), "center": ((B, 2), torch.float32),
              "keypoints_scoremap": ((B, 256, 256, 21), torch.float32), "keypoint_coord3d": ((B, 21, 3), torch.float32),
              "keypoints_uv": ((B, 21, 2), torch.int32), "hand_mask": ((B, H, W), torch.uint8)}
    for byte in PATTERNS[1:]:
        o = {k: _canaried(*v) for k, v in shapes.items()}
        ctx.fill_scratch(byte)
        _lib.check(ctx.lib.h3d_pipeline_forward(
            ctx.h, p(img), p(hs), B, H, W, 1, None, None, p(o["hand_scoremap"]), p(o["image_crop"]), p(o["scale_crop"]), p(o["center"]),
            p(o["keypoints_scoremap"]), p(o["keypoint_coord3d"]), p(o["keypoints_uv"]), p(o["hand_mask"]), st()), "h3d_pipeline_forward")
        torch.cuda.synchronize()
        _assert_overwritten(o, want, "pipeline after a 0x%02X fill:" % byte)
    # track steps start from the state a detect step leaves, so that the track step crops where the hand is
    base = runtime.TrackState(B, ctx.device)
    ctx.track_step(img, hs, base, True, margin=1.5)
    track_keys = ("image_crop", "scale_crop", "center", "keypoints_scoremap", "keypoint_coord3d", "keypoints_uv")
    for detect in (1, 0):
        ref_state = runtime.TrackState(B, ctx.device)
        ref_state.buffer.copy_(base.buffer)
        ctx.fill_scratch(0x00)
        want = _snap(ctx.track_step(img, hs, ref_state, bool(detect), margin=1.5))
        for byte in PATTERNS[1:]:
            state = runtime.TrackState(B, ctx.device)
            state.buffer.copy_(base.buffer)
            o = {k: _canaried(*shapes[k]) for k in track_keys}
            ctx.fill_scratch(byte)
            _lib.check(ctx.lib.h3d_track_step(
                ctx.h, p(img), p(hs), B, H, W, 1, detect, C.c_float(1.5), C.c_float(float("nan")), p(state.buffer), p(o["image_crop"]),
                p(o["scale_crop"]), p(o["center"]), p(o["keypoints_scoremap"]), p(o["keypoint_coord3d"]), p(o["keypoints_uv"]), st()),
                "h3d_track_step")
            torch.cuda.synchronize()
            _assert_overwritten(o, want, "track step (detect=%d) after a 0x%02X fill:" % (detect, byte))
            _assert_same_bits(state.buffer, ref_state.buffer, "track state (detect=%d) after a 0x%02X fill" % (detect, byte))
    ctx.check_errors()

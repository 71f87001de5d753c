"""h3d_launch_count against the kernels that actually ran: every kernel-launching C entry, and every stage plan shape, is called once
outside the profiler (plans built, frame plans uploaded) and once under torch.profiler; the count's delta must equal the number of
CUDA kernel events of the library (every kernel lives in namespace h3d; the filter drops torch's own kernels and memory sets and
copies).  The profiled calls run in a child process, so that no profiler session runs in the suite's own process (see
test_gpu_conv_direct_paths.py::test_dispatch)."""
import ctypes as C
import json
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(HERE, "golden"))

from hand3d_b200 import _lib  # noqa: E402
import synth_records as SR  # noqa: E402

f32 = np.float32

# C entries that enqueue no kernel, or that this one-process test cannot run
EXCLUDED = {
    "h3d_last_error": "host only", "h3d_version": "host only", "h3d_device_available": "device query",
    "h3d_create": "creates the context (memory sets only)", "h3d_destroy": "frees the context",
    "h3d_set_precision": "configuration", "h3d_get_precision": "configuration", "h3d_set_tuning": "configuration",
    "h3d_check_errors": "reads the error word on the host", "h3d_launch_count": "the count itself",
    "h3d_profile_begin": "configuration", "h3d_profile_end": "synchronises and reads events",
    "h3d_load_weight": "host-to-device copies", "h3d_scope_ready": "host only", "h3d_workspace_bytes": "size query",
    "h3d_set_workspace": "configuration", "h3d_fill_scratch": "memory sets only", "h3d_track_state_bytes": "size query",
    "h3d_pack_conv_weights": "packs on the host and copies", "h3d_free_packed_conv": "frees",
    "h3d_conv2d_tc_geometry": "host only", "h3d_conv2d_wgrad_geometry": "host only", "h3d_conv2d_f32_geometry": "host only",
    "h3d_fully_connected_f32_geometry": "host only", "h3d_eval_store_bytes": "size query",
    "h3d_set_dropout": "configuration (a memory set)", "h3d_dropout_draw": "returns a pointer",
    "h3d_gather_records_p2p": "waits for the records of peer ranks: needs one process per GPU (test_gpu_multi.py)",
}


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _rand(*shape, seed=0, lo=-1.0, hi=1.0):
    return _cu(np.random.default_rng(seed).uniform(lo, hi, shape).astype(f32))


def _lifting_weights(bottleneck):
    from hand3d_b200 import weights as Wt
    return {k: v for k, v in Wt.synthetic_weights(0, bottleneck=bottleneck).items() if k.startswith(("PosePrior", "ViewpointNet"))}


# ------------------------------------------------------------------------------------------------------------ the table
# A case is (id, C entries it reaches, setup): setup(ctx) prepares inputs and switches and returns (run, cleanup or None).
CASES = []


def case(cid, entries):
    def deco(fn):
        CASES.append((cid, tuple(entries), fn))
        return fn
    return deco


def _precision(ctx, p):
    ctx.set_precision(p)


def _tuning(ctx, key, value):
    ctx.set_tuning(key, value)
    return lambda: ctx.set_tuning(key, {"fc_chain": 1, "pdl": 1}.get(key, 0))


for _p in ("bf16x3", "fp16", "fp16_f8c", "fp32_ffma"):
    def _seg(ctx, p=_p):
        _precision(ctx, p)
        img = _rand(2, 64, 64, 3, seed=1, lo=-0.5, hi=0.5)
        return (lambda: ctx.handsegnet(img)), None

    def _pose(ctx, p=_p):
        _precision(ctx, p)
        crop = _rand(2, 64, 64, 3, seed=2, lo=-0.5, hi=0.5)
        return (lambda: ctx.posenet(crop)), None

    def _pipe(ctx, p=_p):
        _precision(ctx, p)
        img, hs = _rand(2, 128, 128, 3, seed=3, lo=-0.5, hi=0.5), _cu(np.array([[1, 0], [0, 1]], f32))
        return (lambda: ctx.pipeline(img, hs, True)), None

    case("handsegnet-" + _p, ["h3d_handsegnet_forward"])(_seg)
    case("posenet-" + _p, ["h3d_posenet_forward"])(_pose)
    case("pipeline-" + _p, ["h3d_pipeline_forward"])(_pipe)

for _p in ("bf16x3", "fp32_ffma"):
    for _v in ("proposed", "direct", "bottleneck", "local"):
        for _drop in (False, True):
            for _chain in ((0, 1) if _p == "bf16x3" else (1,)):
                def _lift(ctx, p=_p, v=_v, drop=_drop, chain=_chain):
                    _precision(ctx, p)
                    ctx.load_weights(_lifting_weights(v == "bottleneck"))
                    undo = _tuning(ctx, "fc_chain", chain)
                    sm, hs = _rand(3, 32, 32, 21, seed=4, lo=0.0, hi=1.0), _cu(np.array([[1, 0], [0, 1], [1, 0]], f32))

                    def cleanup():
                        undo()
                        ctx.load_weights(_lifting_weights(False))
                    return (lambda: ctx.lifting(sm, hs, v, dropout=drop)), cleanup
                case("lifting-%s-%s-drop%d-chain%d" % (_p, _v, _drop, _chain), ["h3d_lifting_forward"])(_lift)

for _key in ("no_seg_fusion", "no_pool_fusion", "c3_ffma"):
    def _switched(ctx, key=_key):
        _precision(ctx, "bf16x3")
        undo = _tuning(ctx, key, 1)
        img, hs = _rand(2, 128, 128, 3, seed=5, lo=-0.5, hi=0.5), _cu(np.array([[1, 0], [0, 1]], f32))
        return (lambda: ctx.pipeline(img, hs, True)), undo
    case("pipeline-" + _key, ["h3d_pipeline_forward"])(_switched)


@case("pipeline-2d-no-keypoints", ["h3d_pipeline_forward"])
def _pipe_no_kp(ctx):
    from hand3d_b200.runtime import _ptr, _stream
    _precision(ctx, "bf16x3")
    img = _rand(2, 128, 128, 3, seed=6, lo=-0.5, hi=0.5)
    ctx.ensure_workspace(2, 128, 128)
    N = None

    def run():
        _lib.check(ctx.lib.h3d_pipeline_forward(ctx.h, _ptr(img), N, 2, 128, 128, 0, N, N, N, N, N, N, N, N, N, N, _stream()), "pipeline")
    return run, None


@case("pipeline-2d-keypoints", ["h3d_pipeline_forward"])
def _pipe_2d(ctx):
    _precision(ctx, "bf16x3")
    img = _rand(2, 128, 128, 3, seed=6, lo=-0.5, hi=0.5)
    return (lambda: ctx.pipeline(img, None, False, outputs="keypoints")), None


@case("pose2d-keypoints", ["h3d_pose2d_forward"])
def _pose2d(ctx):
    _precision(ctx, "bf16x3")
    crop = _rand(2, 64, 64, 3, seed=7, lo=-0.5, hi=0.5)
    return (lambda: ctx.pose2d(crop)), None


@case("pose2d-no-keypoints", ["h3d_pose2d_forward"])
def _pose2d_no_kp(ctx):
    from hand3d_b200.runtime import _ptr, _stream
    _precision(ctx, "bf16x3")
    crop = _rand(2, 64, 64, 3, seed=7, lo=-0.5, hi=0.5)
    sm = torch.empty((2, 64, 64, 21), dtype=torch.float32, device="cuda")
    ctx.ensure_workspace(2, 8, 8)
    return (lambda: _lib.check(ctx.lib.h3d_pose2d_forward(ctx.h, _ptr(crop), 2, 64, 64, _ptr(sm), None, _stream()), "pose2d")), None


def _track_inputs(B):
    from hand3d_b200 import runtime
    from hand3d_b200 import weights as Wt
    img = _cu(Wt.synthetic_blob_images(B, 128, 128, seed=8))
    hs = _cu(Wt.synthetic_hand_side(B, seed=9))
    return img, hs, runtime.TrackState(B)


for _detect in (True, False):
    def _track(ctx, detect=_detect):
        _precision(ctx, "bf16x3")
        img, hs, st = _track_inputs(3)
        return (lambda: ctx.track_step(img, hs, st, detect)), None
    case("track-step-detect%d" % _detect, ["h3d_track_step"])(_track)

for _n in (0, 1, 3):
    def _slots(ctx, n=_n):
        _precision(ctx, "bf16x3")
        img, hs, st = _track_inputs(3)
        lost = _cu(np.array([1 if b < n else 0 for b in range(3)], np.int32))

        def run():
            st.lost.copy_(lost)
            ctx.track_step_slots(img, hs, st, outputs="keypoints")
        return run, None
    case("track-step-slots-n%d" % _n, ["h3d_track_step_slots"])(_slots)


@case("track-update", ["h3d_track_update"])
def _track_update(ctx):
    from hand3d_b200 import runtime
    st = runtime.TrackState(2)
    sm = _rand(2, 32, 32, 21, seed=10, lo=0.0, hi=1.0)
    uv = _cu(np.random.default_rng(11).integers(0, 32, (2, 21, 2)).astype(np.int32))
    cen, scl = _cu(np.full((2, 2), 100, f32)), _cu(np.ones(2, f32))
    return (lambda: ctx.track_update(sm, uv, cen, scl, st)), None


for _name, _shape in (("splitk", (1, 8, 8, 64, 64)), ("nosplit", (1, 160, 160, 8, 8))):
    def _conv_f32(ctx, shape=_shape):
        B, H, W, Cin, Cout = shape
        x, w, b = _rand(B, H, W, Cin, seed=12), _rand(3, 3, Cin, Cout, seed=13), _rand(Cout, seed=14)
        return (lambda: ctx.conv2d(x, w, b)), None
    case("conv2d-f32-" + _name, ["h3d_conv2d_f32"])(_conv_f32)

for _p in ("bf16x3", "fp16", "fp16_f8c"):
    def _conv_tc(ctx, p=_p):
        x = _rand(1, 16, 16, 64, seed=15)
        w, b = np.random.default_rng(16).uniform(-1, 1, (3, 3, 64, 64)).astype(f32), np.zeros(64, f32)
        return (lambda: ctx.conv2d_tc(x, w, b, precision=p, stride=2)), None

    def _conv_packed(ctx, p=_p):
        x = _rand(1, 16, 16, 64, seed=15)
        w, b = np.random.default_rng(16).uniform(-1, 1, (3, 3, 64, 64)).astype(f32), np.zeros(64, f32)
        pk = ctx.pack_conv(w, b, precision=p)
        return (lambda: ctx.conv2d_tc_packed(x, pk)), None

    def _conv_layer(ctx, p=_p):
        x = _rand(1, 16, 16, 64, seed=15)
        w, b = np.random.default_rng(16).uniform(-1, 1, (3, 3, 64, 64)).astype(f32), np.zeros(64, f32)
        return (lambda: ctx.conv_layer(x, w, b, p, route=0, pool=1)), None

    case("conv2d-tc-strided-" + _p, ["h3d_conv2d_tc_strided"])(_conv_tc)
    case("conv2d-tc-packed-" + _p, ["h3d_conv2d_tc_packed"])(_conv_packed)
    case("conv-layer-planes-route0-" + _p, ["h3d_conv2d_layer_planes"])(_conv_layer)


@case("conv2d-tc", ["h3d_conv2d_tc"])
def _conv_tc_plain(ctx):
    from hand3d_b200.runtime import _ptr, _stream
    x, y = _rand(1, 16, 16, 64, seed=15), torch.empty((1, 16, 16, 64), dtype=torch.float32, device="cuda")
    w, b = np.random.default_rng(16).uniform(-1, 1, (3, 3, 64, 64)).astype(f32), np.zeros(64, f32)
    return (lambda: _lib.check(ctx.lib.h3d_conv2d_tc(ctx.h, _ptr(x), w.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), _ptr(y),
                                                     1, 16, 16, 64, 64, 3, 1, _lib.PREC_BF16X3, _stream()), "conv2d_tc")), None


@case("conv-layer-planes-route1", ["h3d_conv2d_layer_planes"])
def _conv_layer_direct(ctx):
    x = _rand(1, 16, 16, 3, seed=17)
    w, b = np.random.default_rng(18).uniform(-1, 1, (3, 3, 3, 64)).astype(f32), np.zeros(64, f32)
    return (lambda: ctx.conv_layer(x, w, b, "bf16x3", route=1)), None


for _p in ("bf16x3", "fp16"):
    for _stride in (1, 2):
        def _conv_dev(ctx, p=_p, stride=_stride):
            x, w, b = _rand(1, 16, 16, 64, seed=19), _rand(3, 3, 64, 64, seed=20), _rand(64, seed=21)
            return (lambda: ctx.conv2d_tc_dev(x, w, b, stride=stride, precision=p)), None
        case("conv2d-tc-dev-%s-s%d" % (_p, _stride), ["h3d_conv2d_tc_dev"])(_conv_dev)

for _dx in (False, True):
    for _dw in (False, True):
        for _db in (False, True):
            def _backward(ctx, dx=_dx, dw=_dw, db=_db):
                x, w = _rand(1, 16, 16, 64, seed=22), _rand(3, 3, 64, 32, seed=23)
                y, dy = _rand(1, 8, 8, 32, seed=24), _rand(1, 8, 8, 32, seed=25)
                return (lambda: ctx.conv2d_tc_backward(x, y, dy, w, stride=2, leaky=True, need_dx=dx, need_dw=dw, need_db=db)), None
            case("conv2d-tc-backward-dx%d-dw%d-db%d" % (_dx, _dw, _db), ["h3d_conv2d_tc_backward"])(_backward)

for _H in (512, 520):
    def _seg_post(ctx, H=_H):
        logits = _rand(1, H, 96, 2, seed=26, lo=-3.0, hi=3.0)
        return (lambda: ctx.seg_postprocess(logits)), None
    case("seg-postprocess-%d" % _H, ["h3d_seg_postprocess"])(_seg_post)


@case("frames", ["h3d_resize_frames", "h3d_resize_frames_fmt", "h3d_convert_frames"])
def _frames(ctx):
    from hand3d_b200.runtime import _ptr, _stream
    rgb = _cu(np.random.default_rng(27).integers(0, 256, (2, 60, 80, 3), dtype=np.uint8))
    nv12 = _cu(np.random.default_rng(28).integers(0, 256, (2, 60 * 3 // 2, 80), dtype=np.uint8))
    out = torch.empty((2, 32, 32, 3), dtype=torch.float32, device="cuda")

    def run():
        _lib.check(ctx.lib.h3d_resize_frames(ctx.h, _ptr(rgb), 2, 60, 80, 32, 32, 1, _ptr(out), _stream()), "resize_frames")
        ctx.resize_frames(nv12, 32, 32, False, pixel_format="nv12")
        ctx.convert_frames(nv12, "nv12")
    return run, None


@case("reader", ["h3d_decode_records", "h3d_decode_records_gather", "h3d_reader_next_serials", "h3d_rhd_reader_items",
                 "h3d_stb_reader_items", "h3d_gaussian_scoremap", "h3d_reader_aug_params", "h3d_augment_image",
                 "h3d_rhd_reader_items_aug", "h3d_gaussian_scoremap_dropout", "h3d_canonical_trafo"])
def _reader(ctx):
    rhd = _cu(np.frombuffer(b"".join(SR.rhd_records(4)), np.uint8).reshape(4, -1).copy())
    stb = _cu(np.frombuffer(b"".join(SR.stb_records(2)), np.uint8).reshape(2, -1).copy())
    state = torch.zeros(_lib.READER_STATE_WORDS, dtype=torch.int64, device="cuda")
    serials = _cu(np.array([0, 3, 1, 2], np.int64))
    coords, vis = _rand(4, 21, 2, seed=29, lo=0.0, hi=64.0), _cu(np.ones((4, 21), np.uint8))
    xyz = _rand(4, 21, 3, seed=30)

    def run():
        raw = ctx.decode_records(rhd, "rhd", 1)
        ctx.decode_records_gather(rhd, serials, "rhd", 2)
        st = ctx.decode_records(stb, "stb", 1)
        ctx.reader_next_serials(state, 4, 5, True)
        ctx.rhd_reader_items(raw["header"], raw["mask"], raw["visibility"], True, True, 256)
        ctx.stb_reader_items(st["header"])
        ctx.gaussian_scoremap(coords, (64, 64), 25.0, vis)
        params = ctx.reader_aug_params(serials, 5, 127)
        ctx.augment_image(raw["image"], params, _lib.AUG_HUE | _lib.AUG_RANDOM_CROP, raw["mask"])
        ctx.rhd_reader_items_aug(raw["header"], raw["mask"], raw["visibility"], params, _lib.AUG_COORD_UV_NOISE, True, True, 256)
        ctx.gaussian_scoremap_dropout(coords, (64, 64), 25.0, vis, params[:, _lib.AUG_KEEP:_lib.AUG_KEEP + 21], 0.8)
        ctx.canonical_trafo(xyz)
    return run, None


@case("eval", ["h3d_eval_keypoint_dist", "h3d_eval_feed", "h3d_eval_stats"])
def _eval(ctx):
    gt, pred = _rand(5, 21, 2, seed=31), _rand(5, 21, 2, seed=32)
    vis = _cu(np.ones((5, 21), np.uint8))
    code = _lib.EVAL_FLOAT32
    store = torch.zeros(int(ctx.lib.h3d_eval_store_bytes(21, 64, code)), dtype=torch.uint8, device="cuda")
    thr = _cu(np.linspace(0.0, 1.0, 10))

    def run():
        ctx.eval_keypoint_dist(gt, vis, pred)
        ctx.eval_feed(store, 21, 64, gt, vis, pred)
        ctx.eval_stats(store, 21, 64, torch.float32, thr)
    return run, None


@case("draw", ["h3d_draw_segments"])
def _draw(ctx):
    img = torch.zeros((2, 64, 64, 3), dtype=torch.uint8, device="cuda")
    seg = _rand(2, 3, 4, seed=33, lo=0.0, hi=63.0)
    cols = np.array([[255, 0, 0], [0, 255, 0], [0, 0, 255]], f32)
    return (lambda: ctx.draw_segments(img, seg, cols, 2.0)), None


@case("dropout", ["h3d_dropout_forward", "h3d_dropout_forward_planes", "h3d_dropout_backward", "h3d_dropout_advance"])
def _dropout(ctx):
    from hand3d_b200.runtime import _ptr, _stream
    x = _rand(8, 100, seed=34)
    hi = torch.empty((8, 128), dtype=torch.int16, device="cuda")
    lo = torch.empty((8, 128), dtype=torch.int16, device="cuda")

    def run():
        y, keep = ctx.dropout_forward(x, 0.8, _lib.DROPOUT_LAYER_OP)
        _lib.check(ctx.lib.h3d_dropout_forward_planes(ctx.h, _ptr(x), 8, 100, C.c_float(0.8), _lib.DROPOUT_LAYER_OP, None, None, 0, 128,
                                                      _ptr(hi), _ptr(lo), _stream()), "dropout_forward_planes")
        ctx.dropout_backward(y, keep, 0.8)
        ctx.dropout_advance()
    return run, None


@case("training", ["h3d_resize_bilinear_tf1_backward", "h3d_scoremap_loss_forward", "h3d_scoremap_loss_backward",
                   "h3d_softmax_xent_forward", "h3d_softmax_xent_backward", "h3d_adam_state_set", "h3d_adam_set_lr", "h3d_adam_step"])
def _training(ctx):
    from hand3d_b200 import optim
    dy = _rand(2, 16, 24, 21, seed=35)
    pred, target, vis = _rand(2, 16, 16, 21, seed=36), _rand(2, 16, 16, 21, seed=37), _cu(np.ones((2, 21), f32))
    logits, labels = _rand(2, 8, 8, 2, seed=38), _rand(2, 8, 8, 2, seed=39, lo=0.0, hi=1.0)
    p = torch.nn.Parameter(_rand(300, seed=40))
    p.grad = _rand(300, seed=41)

    def run():
        ctx.resize_bilinear_backward(dy, 8, 8)         # both dimensions change: two kernels
        ctx.resize_bilinear_backward(dy, 16, 8)        # one dimension: one kernel
        ctx.resize_bilinear_backward(dy, 16, 24)       # none: a copy
        _, rms = ctx.scoremap_loss(pred, target, vis)
        ctx.scoremap_loss_backward(pred, target, vis, rms)
        ctx.softmax_xent(logits, labels)
        ctx.softmax_xent_backward(logits, labels)
        opt = optim.Adam([p], 1e-3)                    # h3d_adam_state_set
        opt.set_lr(1e-4)
        opt.step()
    return run, None


@case("lifting-ops", ["h3d_rotate_canonical_backward", "h3d_bone_rel_trafo_inv_backward", "h3d_bone_rel_trafo", "h3d_mse_loss_forward",
                      "h3d_mse_loss_backward", "h3d_bone_rel_trafo_inv", "h3d_rotate_canonical", "h3d_flip_right_hand"])
def _lifting_ops(ctx):
    can, uxyz, hs = _rand(2, 21, 3, seed=42), _rand(2, 3, seed=43), _cu(np.array([[1, 0], [0, 1]], f32))
    d_out = _rand(2, 21, 3, seed=44)
    cond = _cu(np.array([1, 0], np.uint8))

    def run():
        ctx.rotate_canonical_backward(can, uxyz, hs, d_out, None)
        ctx.bone_rel_trafo_inv_backward(can, d_out)
        ctx.bone_rel_trafo(can)
        ctx.mse_loss(can, d_out)
        ctx.mse_loss_backward(can, d_out)
        ctx.bone_rel_trafo_inv(can)
        ctx.rotate_canonical(can, uxyz, hs)
        ctx.flip_right_hand(can, cond)
    return run, None


@case("operators", ["h3d_leaky_relu_f32", "h3d_maxpool2x2_f32", "h3d_maxpool2x2_backward_f32", "h3d_fully_connected_f32",
                    "h3d_resize_bilinear_tf1", "h3d_avgpool8", "h3d_calc_center_bb", "h3d_crop_image_from_xy", "h3d_detect_keypoints",
                    "h3d_upsample_detect_keypoints", "h3d_pack_records"])
def _operators(ctx):
    x, dy = _rand(2, 16, 16, 8, seed=45), _rand(2, 8, 8, 8, seed=46)
    fx, fw, fb = _rand(4, 64, seed=47), _rand(64, 32, seed=48), _rand(32, seed=49)
    mask = _cu((np.random.default_rng(50).uniform(0, 1, (2, 32, 32)) > 0.5).astype(f32))
    img = _rand(2, 64, 64, 3, seed=51)
    cen, scale = _cu(np.full((2, 2), 32, f32)), _cu(np.ones(2, f32))
    sm = _rand(2, 32, 32, 21, seed=52, lo=0.0, hi=1.0)
    c3, uv = _rand(2, 21, 3, seed=53), _cu(np.zeros((2, 21, 2), np.int32))

    def run():
        ctx.leaky_relu(x)
        ctx.max_pool(x)
        ctx.max_pool_backward(x, dy)
        ctx.fully_connected(fx, fw, fb)
        ctx.resize_bilinear(x, 32, 32)
        ctx.avg_pool8(x)
        ctx.calc_center_bb(mask)
        ctx.crop_image_from_xy(img, cen, 32, scale)
        ctx.detect_keypoints(sm)
        ctx.upsample_detect_keypoints(sm, 256, 256)
        ctx.pack_records(c3, uv, cen, scale.reshape(2, 1))
    return run, None


# ------------------------------------------------------------------------------------------------------------ checks
def test_every_entry_is_covered():
    """Every C entry is in the table or excluded with a reason, so that a new entry cannot skip the check."""
    covered = {e for _, entries, _ in CASES for e in entries}
    assert not covered & set(EXCLUDED), covered & set(EXCLUDED)
    missing = sorted(set(_lib.SIGNATURES) - covered - set(EXCLUDED))
    assert not missing, "entries neither in CASES nor in EXCLUDED: %s" % missing
    unknown = sorted((covered | set(EXCLUDED)) - set(_lib.SIGNATURES))
    assert not unknown, unknown
    assert len({cid for cid, _, _ in CASES}) == len(CASES)


def run_cases(path):
    """The child: each case once outside and once inside a profiler session; writes {id: {launches, kernels}} as JSON."""
    from torch.profiler import ProfilerActivity, profile
    from hand3d_b200 import runtime
    from hand3d_b200 import weights as Wt
    ctx = runtime.default_context()
    ctx.load_weights(Wt.synthetic_weights(0))
    ctx.set_dropout(5)

    def profiled(fn):
        """(launch-count delta, the library's kernel names) of one call of fn under a profiler session.  A session that recorded no CUDA
        event at all (the first session of a process sometimes misses its kernels) is repeated once."""
        for _ in range(2):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                n0 = ctx.launch_count
                fn()
                torch.cuda.synchronize()
                n1 = ctx.launch_count
            cuda = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
            if cuda or n1 == n0:
                break
        return n1 - n0, [n for n in cuda if "h3d::" in n]

    profiled(lambda: torch.ones(1, device="cuda").add_(1))  # a first session on torch's own kernel
    out = {}
    for cid, _, setup in CASES:
        try:
            run, cleanup = setup(ctx)
            run()                                           # warm-up: plans, packed weights, frame plans
            torch.cuda.synchronize()
            launches, names = profiled(run)
            if cleanup:
                cleanup()
        except Exception as e:                              # reported by the case's test; the other cases still run
            out[cid] = {"error": "%s: %s" % (type(e).__name__, e)}
            print("%-44s %s" % (cid, out[cid]["error"]), flush=True)
            continue
        out[cid] = {"launches": launches, "kernels": names}
        print("%-44s launches %3d kernels %3d" % (cid, launches, len(names)), flush=True)
    ctx.set_dropout(None)
    torch.cuda.synchronize()
    ctx.check_errors()
    with open(path, "w") as f:
        json.dump(out, f)


@pytest.fixture(scope="module")
def counted(tmp_path_factory):
    import subprocess
    path = str(tmp_path_factory.mktemp("launch_count") / "counts.json")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), path], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=1200)
    assert r.returncode == 0, "launch-count child failed:\n" + r.stdout[-6000:]
    with open(path) as f:
        return json.load(f)


@pytest.mark.gpu
@pytest.mark.parametrize("cid", [cid for cid, _, _ in CASES])
def test_launch_count_equals_kernels_run(counted, cid):
    got = counted[cid]
    assert "error" not in got, got.get("error")
    assert got["launches"] == len(got["kernels"]), "%s: h3d_launch_count moved by %d, the profiler saw %d kernels:\n%s" % (
        cid, got["launches"], len(got["kernels"]), "\n".join(got["kernels"]))
    assert got["launches"] > 0 or cid.startswith("conv2d-tc-backward-dx0-dw0-db0"), cid


if __name__ == "__main__" and len(sys.argv) == 2:
    run_cases(sys.argv[1])

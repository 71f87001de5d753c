"""Images above 512 px a side, up to H3D_PIPELINE_MAX_SIDE = 2048: the thread-block-cluster mask grower bit for bit against the
reference's single_obj_scoremap / calc_center_bb, its dispatch, the pipeline at these sizes (parity, batches whose activation planes
pass 2^31 bytes, CUDA graphs) and the refusal of larger images.

Everything runs in a private Context: at 1080x1920 with B = 9 its workspace is many GB, which must not stay allocated in the process's
default context for the test modules that follow."""
import gc

import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import grow_oracle as G
from hand3d_b200 import _lib
from hand3d_b200 import weights as Wt
from oracle import hand3d_oracle as O
from oracle import tf1_ops as T

pytestmark = pytest.mark.gpu
W_SEG = Wt.synthetic_weights(0, seg_shift=0.15)   # blob images give varied masks with these


@pytest.fixture(scope="module")
def ctx():
    from hand3d_b200 import runtime
    c = runtime.Context()
    try:
        c.load_weights(W_SEG)
        c.set_precision("bf16x3")
        yield c
    finally:
        torch.cuda.synchronize()
        c.release_graphs()
        c.lib.h3d_destroy(c.h)
        c.h = None
        c._ws = None
        del c
        gc.collect()
        torch.cuda.empty_cache()


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _host(r):
    return {k: v.cpu().numpy() for k, v in r.items() if v is not None}


GROW_SHAPES = [(513, 513), (480, 640), (640, 480), (720, 1280), (1080, 1920), (2048, 2048), (17, 2048), (2048, 17),
               (600, 1000), (531, 777), (1499, 999), (33, 1025)]   # the last four: widths that are not multiples of 32


@pytest.mark.parametrize("H,W", GROW_SHAPES)
def test_grower_bit_exact(ctx, H, W):
    cases = [G.make_case(H, W, k, seed=H + W + i) for i, k in enumerate(G.KINDS)]
    logits = G.logits_of(cases)
    ref = G.seg_postprocess(logits)
    got = _host(ctx.seg_postprocess(_dev(logits)))
    for k in ("max_loc", "hand_mask", "center", "crop_size", "scale_crop"):
        np.testing.assert_array_equal(got[k], ref[k], err_msg="%s at %dx%d" % (k, H, W))
    serp = G.KINDS.index("serpentine")
    assert 0 < got["hand_mask"][serp].sum() < cases[serp][0].sum(), "the pass count must truncate the corridor"
    # B = 1 and B = 5: each image equals its row of the batch
    got5 = _host(ctx.seg_postprocess(_dev(logits[:5])))
    for k in got5:
        np.testing.assert_array_equal(got5[k], got[k][:5], err_msg=k)
    for b in (0, 3, 6):
        got1 = _host(ctx.seg_postprocess(_dev(logits[b:b + 1])))
        for k in got1:
            np.testing.assert_array_equal(got1[k], got[k][b:b + 1], err_msg="%s, image %d" % (k, b))


def _kernels(fn):
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def test_dispatch(ctx):
    """512 a side still runs the single-CTA mask_grow_kernel; one pixel more on either side runs the cluster kernel."""
    for (H, W), name in [((512, 512), "mask_grow_kernel"), ((513, 512), "mask_grow_cluster_kernel"), ((512, 513), "mask_grow_cluster_kernel")]:
        logits = _dev(G.logits_of([G.make_case(H, W, "blobs", 1)]))
        ctx.seg_postprocess(logits)   # warm-up outside the profiler
        names = _kernels(lambda: ctx.seg_postprocess(logits))
        grow = [n for n in names if "mask_grow" in n]
        assert len(grow) == 1, (H, W, names)
        assert ("mask_grow_cluster_kernel" in grow[0]) == (name == "mask_grow_cluster_kernel") and name in grow[0], (H, W, grow)


def test_pipeline_hand_scoremap_520x1040(ctx):
    B, H, W = 2, 520, 1040
    img = Wt.synthetic_blob_images(B, H, W, seed=7)
    hs = Wt.synthetic_hand_side(B, seed=8)
    g = _host(ctx.pipeline(_dev(img), _dev(hs), True, want_mask=True))
    ref = O.inference_detection(img, W_SEG)[-1]
    err = np.abs(g["hand_scoremap"] - ref).max()
    print("520x1040 hand_scoremap: max abs err %.2e" % err)
    assert err < 1e-3


@pytest.mark.parametrize("H,W", [(480, 640), (1080, 1920)])
def test_pipeline_teacher_forced(ctx, H, W):
    """Every stage against the oracle fed with the device's own outputs of the stage before."""
    B = 2
    img = Wt.synthetic_blob_images(B, H, W, seed=H)
    hs = Wt.synthetic_hand_side(B, seed=W)
    g = _host(ctx.pipeline(_dev(img), _dev(hs), True, want_mask=True))
    # mask, centre and scale: exact functions of the device's logits
    ref = G.seg_postprocess(g["hand_scoremap"])
    np.testing.assert_array_equal(g["hand_mask"], ref["hand_mask"])
    np.testing.assert_array_equal(g["center"], ref["center"])
    np.testing.assert_array_equal(g["scale_crop"], ref["scale_crop"])
    assert ref["hand_mask"].reshape(B, -1).sum(1).min() > 0, "the blob images are meant to give a hand mask"
    # crop
    crop = O.crop_image_from_xy(img, g["center"], 256, g["scale_crop"])
    assert np.abs(g["image_crop"] - crop).max() < 1e-3
    # PoseNet, up-sampling, key-points, lifting on the device's crop
    s32 = O.inference_pose2d(g["image_crop"], W_SEG)[-1]
    kp_map = T.resize_bilinear_tf1(s32.astype(np.float32), 256, 256)
    assert np.abs(g["keypoints_scoremap"] - kp_map).max() < 1e-3
    for b in range(B):
        np.testing.assert_array_equal(g["keypoints_uv"][b], O.detect_keypoints(g["keypoints_scoremap"][b]).astype(np.int32))
        kp_ref = O.detect_keypoints(kp_map[b]).astype(np.int32)
        for c in range(21):   # the oracle's own arg-max: identical unless its map has a near-tie there
            v, u = g["keypoints_uv"][b, c]
            assert (g["keypoints_uv"][b, c] == kp_ref[c]).all() or kp_map[b, :, :, c].max() - kp_map[b, v, u, c] < 2e-3, (b, c)
    coord3d = O.inference_pose3d(s32, hs, W_SEG)[0]
    assert np.abs(g["keypoint_coord3d"] - coord3d).max() < 1e-3


def test_capture_pipeline_1080p_replays_eager(ctx):
    B, H, W = 2, 1080, 1920
    img = _dev(Wt.synthetic_blob_images(B, H, W, seed=11))
    hs = _dev(Wt.synthetic_hand_side(B, seed=12))
    eager = _host(ctx.pipeline(img, hs, True, outputs="keypoints"))
    replay, res = ctx.capture_pipeline(img, hs, True)
    try:
        replay()
        torch.cuda.synchronize()
        got = _host(res)
        for k in eager:
            np.testing.assert_array_equal(got[k], eager[k], err_msg=k)
    finally:
        del replay, res
        ctx.release_graphs()


@pytest.mark.parametrize("H,W", [(2049, 640), (640, 2049), (2049, 2049)])
def test_larger_images_are_refused_before_any_launch(ctx, H, W):
    img = torch.zeros((1, H, W, 3), dtype=torch.float32, device="cuda")
    logits = torch.zeros((1, H, W, 2), dtype=torch.float32, device="cuda")
    out = [torch.zeros(n, dtype=torch.float32, device="cuda") for n in (2, 1, 1)]
    torch.cuda.synchronize()
    n0 = ctx.launch_count
    rc = []

    def calls():
        rc.append(ctx.lib.h3d_pipeline_forward(ctx.h, _lib.C.c_void_p(img.data_ptr()), None, 1, H, W, 0, None, None, None, None,
                                               _lib.C.c_void_p(out[2].data_ptr()), _lib.C.c_void_p(out[0].data_ptr()), None, None, None,
                                               None, None))
        rc.append(ctx.lib.h3d_seg_postprocess(ctx.h, _lib.C.c_void_p(logits.data_ptr()), 1, H, W, None, None,
                                              _lib.C.c_void_p(out[0].data_ptr()), None, _lib.C.c_void_p(out[2].data_ptr()), None))

    names = _kernels(calls)
    assert rc == [_lib.EINVAL, _lib.EINVAL]
    assert "2048" in _lib.last_error()
    assert names == [], names
    assert ctx.launch_count == n0


def test_batch_past_2_31_bytes_per_plane(ctx):
    """1080x1920 with B = 9: one 64-channel 2-byte activation plane holds 9 * 1080 * 1920 * 64 * 2 = 2.39e9 bytes > 2^31.  The first,
    middle and last image equal their own B = 1 runs bit for bit."""
    B, H, W = 9, 1080, 1920
    assert B * H * W * 64 * 2 > 2 ** 31
    need = int(ctx.lib.h3d_workspace_bytes(ctx.h, B, H, W))
    free, _ = torch.cuda.mem_get_info()
    print("h3d_workspace_bytes(B=%d, %dx%d) = %.2f GB, free %.2f GB" % (B, H, W, need / 1e9, free / 1e9))
    inputs = B * H * W * 3 * 4 + B * H * W * (2 * 4 + 1)
    if need + inputs + (1 << 30) > free:
        pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % ((need + inputs) / 1e9, free / 1e9))
    img = Wt.synthetic_blob_images(B, H, W, seed=13)
    hs = Wt.synthetic_hand_side(B, seed=14)
    full = _host(ctx.pipeline(_dev(img), _dev(hs), True, want_mask=True))
    for b in (0, B // 2, B - 1):
        one = _host(ctx.pipeline(_dev(img[b:b + 1]), _dev(hs[b:b + 1]), True, want_mask=True))
        for k in one:
            np.testing.assert_array_equal(one[k], full[k][b:b + 1], err_msg="%s, image %d" % (k, b))

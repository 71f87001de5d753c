"""Size-independent properties checked at BASELINE.json's batch sizes (where the CPU oracle would take minutes):
batch independence (an image's result does not depend on its batch neighbours, on the batch size or on how the
batch is sharded -- the property multi-GPU sharding relies on), determinism, and agreement between precision modes."""
import numpy as np
import pytest
import torch

from hand3d_b200 import weights as Wt

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from hand3d_b200 import runtime
    c = runtime.default_context()
    c.load_weights(Wt.synthetic_weights(0))
    c.set_precision("bf16x3")
    return c


def _run(ctx, img, hs):
    r = ctx.pipeline(torch.from_numpy(img).cuda(), torch.from_numpy(hs).cuda(), True)
    return {k: v.cpu().numpy() for k, v in r.items() if v is not None}


DISCRETE = ["center", "scale_crop", "keypoints_uv", "image_crop"]
CONV = ["hand_scoremap", "keypoints_scoremap"]


def test_batch_independence_and_sharding_b32(ctx):
    """Full batch of 32 (BASELINE config 4 per-GPU shard) == two shards of 16 == ragged shards 7 + 25, bit for bit, 3-D coordinates
    included: in bf16x3 the lifting's pyramids run on conv_tc_kernel, whose arithmetic does not depend on B, and the FC chain computes
    each row on its own (no split-K on the tensor-core path)."""
    B = 32
    img = Wt.synthetic_images(B, 320, 320, seed=21)
    hs = Wt.synthetic_hand_side(B, seed=22)
    full = _run(ctx, img, hs)
    for cuts in ([0, 16, 32], [0, 7, 32], [0, 1, 2, 32]):
        parts = [_run(ctx, img[a:b], hs[a:b]) for a, b in zip(cuts[:-1], cuts[1:])]
        for k in DISCRETE + CONV + ["keypoint_coord3d"]:
            np.testing.assert_array_equal(np.concatenate([p[k] for p in parts], 0), full[k], err_msg="%s, cuts %s" % (k, cuts))


def test_determinism(ctx):
    img = Wt.synthetic_images(5, 320, 320, seed=23)
    hs = Wt.synthetic_hand_side(5, seed=24)
    a, b = _run(ctx, img, hs), _run(ctx, img, hs)
    for k in a:
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)


def test_precision_modes_agree_at_full_size(ctx):
    """B = 16 at 320x320: the three fp32-parity modes agree within 1e-3 of each other with teacher-forced crops
    (fp32_ffma is bit-wise the CUDA-core fp32 yard-stick), and the fp16 mode stays within 1e-2."""
    B = 16
    img = Wt.synthetic_images(B, 320, 320, seed=25)
    hs = Wt.synthetic_hand_side(B, seed=26)
    ti, th = torch.from_numpy(img).cuda(), torch.from_numpy(hs).cuda()
    ctx.set_precision("fp32_ffma")
    base = ctx.pipeline(ti, th, True)
    out = {}
    for prec, tol in (("bf16x3", 1e-3), ("fp16x3", 1e-3), ("fp16", 1e-2)):
        ctx.set_precision(prec)
        r = ctx.pipeline(ti, th, True, force_center=base["center"], force_scale=base["scale_crop"])
        out[prec] = r
        for k in ("hand_scoremap", "keypoints_scoremap", "keypoint_coord3d"):
            err = (r[k] - base[k]).abs().max().item()
            assert err < tol, "%s %s: %.3e" % (prec, k, err)
        assert torch.equal(r["image_crop"], base["image_crop"])
    same = (out["bf16x3"]["keypoints_uv"] == base["keypoints_uv"]).all(dim=2).float().mean().item()
    assert same > 0.99, "key-point agreement with the fp32 path: %.4f" % same
    ctx.set_precision("bf16x3")


def test_single_image_and_odd_batch_shapes(ctx):
    for B, H, W in ((1, 320, 320), (3, 240, 320), (5, 320, 240)):
        img = Wt.synthetic_images(B, H, W, seed=27)
        hs = Wt.synthetic_hand_side(B, seed=28)
        r = _run(ctx, img, hs)
        assert r["hand_scoremap"].shape == (B, H, W, 2) and r["keypoints_scoremap"].shape == (B, 256, 256, 21)
        assert np.isfinite(r["keypoint_coord3d"]).all() and np.isfinite(r["keypoints_scoremap"]).all()
        one = _run(ctx, img[:1], hs[:1])
        for k in DISCRETE + CONV:
            np.testing.assert_array_equal(one[k][0], r[k][0], err_msg=k)


def test_cuda_graph_replay_matches_eager(ctx):
    """The whole forward pass (incl. the branches forked onto the context's side streams) captures into one CUDA graph;
    replays on refreshed inputs are bit-identical to eager calls."""
    B = 4
    imgs = [Wt.synthetic_images(B, 320, 320, seed=31 + i) for i in range(2)]
    hs = Wt.synthetic_hand_side(B, seed=33)
    ti, th = torch.from_numpy(imgs[0]).cuda(), torch.from_numpy(hs).cuda()
    replay, res = ctx.capture_pipeline(ti, th, True, outputs="keypoints")
    try:
        for img in imgs[::-1] + imgs:
            ti.copy_(torch.from_numpy(img))
            replay()
            torch.cuda.synchronize()
            got = {k: v.clone() for k, v in res.items() if v is not None}
            ref = ctx.pipeline(ti, th, True, outputs="keypoints")
            for k in ("keypoints_uv", "keypoint_coord3d", "center", "scale_crop"):
                assert torch.equal(got[k], ref[k]), k
        with pytest.raises(RuntimeError, match="release_graphs"):     # plans (and what graphs point into) are frozen while a graph lives
            ctx.set_tuning("pdl", 1)
    finally:
        del replay
        torch.cuda.synchronize()
        ctx.release_graphs()      # later tests may grow the workspace / switch precision again


@pytest.mark.parametrize("prec", ["bf16x3", "fp16"])
def test_repeated_calls_change_no_bit(ctx, prec):
    """Repeated calls give bit-identical outputs (B = 32 and a ragged B = 7): no result depends on how the overlapping launches of
    a call are scheduled or on state an earlier call left behind."""
    ctx.set_precision(prec)
    try:
        for B in (32, 7):
            img = Wt.synthetic_images(B, 320, 320, seed=41)
            hs = Wt.synthetic_hand_side(B, seed=42)
            base = _run(ctx, img, hs)
            for rep in range(9):
                r = _run(ctx, img, hs)
                for k in base:
                    np.testing.assert_array_equal(r[k], base[k], err_msg="%s (rep %d, B %d)" % (k, rep, B))
    finally:
        ctx.set_precision("bf16x3")

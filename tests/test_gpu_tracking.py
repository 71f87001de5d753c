"""Tracking across camera frames (h3d_track_step, Context.track_step, FrameRunner(track=True)): the update kernel against the numpy
restatement (tests/track_oracle.py) bit for bit, a track step against the teacher-forced pipeline, a detect step against the pipeline,
the launches a track step saves, FrameRunner's detect / track policy on a synthetic sequence, and the argument checks."""
import gc

import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import track_oracle as T
from hand3d_b200 import _lib, runtime
from hand3d_b200 import weights as Wt
from hand3d_b200.frames import FrameRunner

pytestmark = pytest.mark.gpu
W_SEG = Wt.synthetic_weights(0, seg_shift=0.15)   # blob images give varied masks with these
F = np.float32


@pytest.fixture(scope="module")
def ctx():
    c = runtime.Context()
    try:
        c.load_weights(W_SEG)
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
    return {k: v.cpu().numpy() for k, v in r.items() if isinstance(v, torch.Tensor)}


def _state_host(st):
    return {"center": st.center.cpu().numpy(), "scale": st.scale.cpu().numpy(), "score": st.score.cpu().numpy(),
            "lost": st.lost.cpu().numpy()}


def _bits_equal(got, want, what):
    """Bit-equal, except that any NaN equals any NaN (numpy keeps a NaN's payload, the device's arithmetic does not)."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    if got.dtype.kind == "f":
        gn, wn = np.isnan(got), np.isnan(want)
        np.testing.assert_array_equal(gn, wn, err_msg="%s: NaN positions" % what)
        got, want = np.where(gn, 0, got).astype(got.dtype), np.where(wn, 0, want).astype(want.dtype)
        got, want = got.view(np.int32), want.view(np.int32)
    np.testing.assert_array_equal(got, want, err_msg=what)


def _random_case(B, seed):
    """Maps, key-points, centres and scales that reach both scale clamps, zero-size boxes and the fall-backs."""
    rng = np.random.default_rng(seed)
    maps = rng.normal(0, 1, (B, 32, 32, 21)).astype(F) * F(rng.uniform(0.01, 3))
    uv = rng.integers(0, 256, (B, 21, 2)).astype(np.int32)
    center = rng.uniform(-200, 1200, (B, 2)).astype(F)
    scale = np.exp(rng.uniform(np.log(0.05), np.log(20), B)).astype(F)
    for b in range(B):
        kind = b % 8
        if kind == 1:
            uv[b] = rng.integers(0, 256, 2)                        # one pixel: size 0 -> scale 5
        elif kind == 2:
            uv[b] = rng.integers(120, 136, (21, 2))                # a small box: the upper clamp
        elif kind == 3:
            scale[b] = F(0.05)                                     # a huge box: the lower clamp
        elif kind == 4:
            scale[b] = [F(0), F(np.nan), F(np.inf)][b % 3]         # x / 0, NaN, x / inf
        elif kind == 5:
            center[b, b % 2] = [F(np.nan), F(np.inf), F(-np.inf)][b % 3]
        elif kind == 6:
            maps[b, b % 32, 7, b % 21] = np.nan                    # NaN score
        elif kind == 7:
            center[b] = F(3e38)                                    # overflowing extents
    return maps, uv, center, scale


@pytest.mark.parametrize("B", [1, 3, 32, 160])
@pytest.mark.parametrize("margin,min_score", [(1.5, None), (1.25, 0.0), (2.0, "median")])
def test_update_kernel_matches_oracle(ctx, B, margin, min_score):
    maps, uv, center, scale = _random_case(B, seed=B * 7 + int(margin * 4))
    if min_score == "median":
        min_score = float(np.nanmedian([T.score(m) for m in maps]))
    st = runtime.TrackState(B)
    rng = np.random.default_rng(B)
    st.center.copy_(_dev(rng.uniform(0, 300, (B, 2)).astype(F)))
    st.scale.copy_(_dev(rng.uniform(0.5, 2, B).astype(F)))
    want = _state_host(st)
    ctx.track_update(_dev(maps), _dev(uv), _dev(center), _dev(scale), st, margin=margin, min_score=min_score)
    got = _state_host(st)
    T.update(want, maps, uv, center, scale, margin, min_score)
    for k in want:
        _bits_equal(got[k], want[k], k)
    if B >= 32:   # the case mix reaches every branch
        assert want["lost"].any() and not want["lost"].all()
        assert (want["scale"] == F(5)).any() and (want["scale"] == F(0.25)).any()


def _forced_step_case(ctx, precision, H, W, seed):
    ctx.set_precision(precision)
    B = 2
    img = _dev(Wt.synthetic_blob_images(B, H, W, seed=seed))
    hs = _dev(Wt.synthetic_hand_side(B, seed=seed + 1))
    det = _host(ctx.pipeline(img, hs, True))
    st = runtime.TrackState(B)
    # a crop near the detected one, as the previous frame's key-points would give
    st.center.copy_(_dev(det["center"] + F([[3.5, -6.0], [-2.25, 4.0]])))
    st.scale.copy_(_dev(det["scale_crop"].reshape(B) * F(1.125)))
    return B, img, hs, st


@pytest.mark.parametrize("precision", ["bf16x3", "fp16"])
@pytest.mark.parametrize("H,W", [(240, 320), (320, 320), (600, 800)])
def test_track_step_equals_forced_pipeline(ctx, precision, H, W):
    B, img, hs, st = _forced_step_case(ctx, precision, H, W, seed=H + W)
    c, s = st.center.clone(), st.scale.clone()
    before = _state_host(st)
    got = _host(ctx.track_step(img, hs, st, detect=False, margin=1.5, min_score=None))
    after = _state_host(st)
    ref = _host(ctx.pipeline(img, hs, True, force_center=c, force_scale=s.reshape(B, 1)))
    for k in ("image_crop", "keypoints_scoremap", "keypoints_uv", "keypoint_coord3d", "center", "scale_crop"):
        _bits_equal(got[k], ref[k], k)
    # the update in place: the oracle on the step's own map, key-points and crop
    map32 = ctx.posenet(_dev(ref["image_crop"]))[2].cpu().numpy()
    T.update(before, map32, ref["keypoints_uv"], ref["center"], ref["scale_crop"], 1.5, None)
    for k in before:
        _bits_equal(after[k], before[k], k)


@pytest.mark.parametrize("precision", ["bf16x3", "fp16"])
def test_detect_step_equals_pipeline(ctx, precision):
    ctx.set_precision(precision)
    B, H, W = 3, 240, 320
    img = _dev(Wt.synthetic_blob_images(B, H, W, seed=5))
    hs = _dev(Wt.synthetic_hand_side(B, seed=6))
    st = runtime.TrackState(B)
    got = _host(ctx.track_step(img, hs, st, detect=True, margin=1.25, min_score=0.0))
    ref = _host(ctx.pipeline(img, hs, True))
    for k in got:
        _bits_equal(got[k], ref[k], k)
    want = T.new_state(B)
    map32 = ctx.posenet(_dev(ref["image_crop"]))[2].cpu().numpy()
    T.update(want, map32, ref["keypoints_uv"], ref["center"], ref["scale_crop"], 1.25, 0.0)
    got_st = _state_host(st)
    for k in want:
        _bits_equal(got_st[k], want[k], k)


def test_track_step_saves_exactly_the_detection_launches(ctx):
    ctx.set_precision("bf16x3")
    B, H, W = 2, 240, 320
    img = _dev(Wt.synthetic_blob_images(B, H, W, seed=9))
    hs = _dev(Wt.synthetic_hand_side(B, seed=10))
    st = runtime.TrackState(B)
    ctx.track_step(img, hs, st, True)
    ctx.track_step(img, hs, st, False)           # warm-up: plans built

    def launches(fn):
        torch.cuda.synchronize()
        n0 = ctx.launch_count
        fn()
        torch.cuda.synchronize()
        return ctx.launch_count - n0

    det = launches(lambda: ctx.track_step(img, hs, st, True, outputs="keypoints"))
    trk = launches(lambda: ctx.track_step(img, hs, st, False, outputs="keypoints"))
    pipe = launches(lambda: ctx.pipeline(img, hs, True, outputs="keypoints"))
    seg = launches(lambda: ctx.handsegnet(img))                  # its x8 up-sampling is fused into the post-processing in the pipeline
    post = launches(lambda: ctx.seg_postprocess(torch.zeros((B, H, W, 2), dtype=torch.float32, device="cuda")))
    print("launches: detect step %d, track step %d, pipeline %d, HandSegNet %d, mask post-processing %d" % (det, trk, pipe, seg, post))
    assert det == pipe + 1                                        # + the update
    assert det - trk == (seg - 1) + post


def _uint8(img):
    return np.clip(np.round((img + 0.5) * 255.0), 0, 255).astype(np.uint8)


def _sequence(n, noise_at, H=240, W=320):
    """Two streams of a blob image shifted (2, 3) px per frame; stream 0 gets a faint-noise frame at noise_at."""
    base = _uint8(Wt.synthetic_blob_images(2, H, W, seed=21))
    rng = np.random.default_rng(22)
    frames = []
    for t in range(n):
        f = np.stack([np.roll(base[b], (2 * t, 3 * t), axis=(0, 1)) for b in range(2)])
        if t == noise_at:
            f[0] = rng.integers(126, 131, (H, W, 3), dtype=np.uint8)
        frames.append(f)
    return frames


def _run(runner, frames):
    return list(runner.stream(frames))


def test_frame_runner_redetect_every_1_equals_plain(ctx):
    ctx.set_precision("bf16x3")
    frames = _sequence(5, noise_at=2)
    try:
        plain = _run(FrameRunner(ctx, 2, (240, 320)), frames)
        tracked = _run(FrameRunner(ctx, 2, (240, 320), track=True, redetect_every=1, min_score=0.0), frames)
    finally:
        ctx.release_graphs()
    assert len(plain) == len(tracked) == 5
    for t, (p, q) in enumerate(zip(plain, tracked)):
        assert q["detected"] is True
        for k in FrameRunner.RESULT_KEYS:
            _bits_equal(q[k], p[k], "%s at step %d" % (k, t))


def _check_policy_and_crops(res, redetect_every, min_score, margin):
    """Replays the host's detect / track choice and the oracle's crops from the device's own key-points and scores."""
    state = None
    for t, r in enumerate(res):
        lost_2 = res[t - 2]["track_lost"].any() if t >= 2 else False
        want_detect = t == 0 or (redetect_every is not None and t % redetect_every == 0) or bool(lost_2)
        assert r["detected"] == want_detect, (t, r["detected"])
        if not r["detected"]:
            _bits_equal(r["center"], state["center"], "center at step %d" % t)
            _bits_equal(r["scale_crop"].reshape(-1), state["scale"], "scale at step %d" % t)
        if state is None:
            state = T.new_state(len(r["center"]))
        for b in range(len(r["center"])):
            c, s, fb = T.next_crop(r["keypoints_uv"][b], r["center"][b], r["scale_crop"][b, 0], margin)
            lost = fb or (min_score is not None and not (r["track_score"][b] >= F(min_score)))
            assert bool(r["track_lost"][b]) == lost, (t, b)
            if not lost:
                state["center"][b], state["scale"][b] = c, s


def test_synthetic_sequence(ctx):
    ctx.set_precision("bf16x3")
    n, noise_at = 9, 3
    frames = _sequence(n, noise_at)
    try:
        # the scores without a threshold: the faint frame's must lie below every blob frame's
        free = _run(FrameRunner(ctx, 2, (240, 320), track=True, track_margin=1.5), frames)
        _check_policy_and_crops(free, None, None, 1.5)
        sc = np.array([r["track_score"] for r in free])          # [step, stream]
        print("scores:", sc.T)
        others = np.delete(sc.reshape(-1), noise_at * 2)
        assert sc[noise_at, 0] < others.min(), "the faint frame is meant to score lowest"
        min_score = float((sc[noise_at, 0] + others.min()) / 2)
        runs = [_run(FrameRunner(ctx, 2, (240, 320), track=True, min_score=min_score, track_margin=1.5), frames) for _ in range(2)]
    finally:
        ctx.release_graphs()
    res = runs[0]
    _check_policy_and_crops(res, None, min_score, 1.5)
    assert res[noise_at]["track_lost"][0] and not res[noise_at]["track_lost"][1]
    assert [r["detected"] for r in res[:noise_at + 3]] == [True] + [False] * (noise_at + 1) + [True]   # lost at t -> detect at t + 2
    for t, (a, b) in enumerate(zip(runs[0], runs[1])):           # two runs
        for k in a:
            _bits_equal(np.asarray(b[k]), np.asarray(a[k]), "%s at step %d" % (k, t))
    # eager against graph replay: the same steps, enqueued one by one
    st = runtime.TrackState(2)
    hs = _dev(np.array([[1.0, 0.0]] * 2, F))
    for t, f in enumerate(frames):
        image = ctx.resize_frames(_dev(f), 240, 320, normalize=True)
        r = _host(ctx.track_step(image, hs, st, res[t]["detected"], margin=1.5, min_score=min_score, outputs="keypoints"))
        for k in ("keypoints_uv", "keypoint_coord3d", "center", "scale_crop"):
            _bits_equal(r[k], res[t][k], "%s at step %d" % (k, t))
        _bits_equal(st.score.cpu().numpy(), res[t]["track_score"], "score at step %d" % t)
        _bits_equal(st.lost.cpu().numpy() != 0, res[t]["track_lost"], "lost at step %d" % t)


def _kernels(fn):
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def test_bad_arguments_are_refused_before_any_launch(ctx):
    B, H, W = 1, 240, 320
    img = torch.zeros((B, H, W, 3), dtype=torch.float32, device="cuda")
    big = torch.zeros((1, 2049, 64, 3), dtype=torch.float32, device="cuda")
    hs = torch.zeros((B, 2), dtype=torch.float32, device="cuda")
    c3d = torch.zeros((B, 21, 3), dtype=torch.float32, device="cuda")
    st = runtime.TrackState(B)
    P = _lib.C.c_void_p
    nan = float("nan")

    def step(image=img, b=B, h=H, w=W, margin=1.5, min_score=nan, state=st.buffer, pose3d=1, coord=c3d):
        return ctx.lib.h3d_track_step(ctx.h, P(image.data_ptr()), P(hs.data_ptr()), b, h, w, pose3d, 0, margin, min_score,
                                      None if state is None else P(state.data_ptr()), None, None, None, None,
                                      None if coord is None else P(coord.data_ptr()), None, None)

    cases = [dict(margin=0.2), dict(margin=float("inf")), dict(margin=nan), dict(min_score=float("inf")), dict(min_score=-float("inf")),
             dict(state=None), dict(b=0), dict(image=big, h=2049, w=64), dict(h=0), dict(coord=None)]
    torch.cuda.synchronize()
    n0 = ctx.launch_count
    rc = []
    names = _kernels(lambda: [rc.append(step(**c)) for c in cases])
    assert rc == [_lib.EINVAL] * len(cases), rc
    assert names == [], names
    assert ctx.launch_count == n0
    m = torch.zeros((B, 32, 32, 21), dtype=torch.float32, device="cuda")
    uv = torch.zeros((B, 21, 2), dtype=torch.int32, device="cuda")
    z = torch.zeros(2, dtype=torch.float32, device="cuda")
    assert ctx.lib.h3d_track_update(ctx.h, P(m.data_ptr()), P(uv.data_ptr()), P(z.data_ptr()), P(z.data_ptr()), B, 0.1, nan,
                                    P(st.buffer.data_ptr()), None) == _lib.EINVAL
    assert ctx.lib.h3d_track_state_bytes(0) == _lib.EINVAL
    assert ctx.lib.h3d_track_state_bytes(3) == 3 * 5 * 4

"""Drawing on the device (h3d_draw_segments, Context.draw_segments, hand3d_b200.draw, FrameRunner(draw=True)): the kernel against the
numpy restatement of its rule (tests/draw_oracle.py) bit for bit over whole images, draw_hand / draw_hand_3d / run_figure's panels,
poisoned scratch, graph capture, argument refusals, and the frame graphs' drawn frames."""
import ctypes as C

import numpy as np
import pytest
import torch

import draw_oracle as O
from hand3d_b200 import _lib, runtime
from hand3d_b200 import draw as D
from hand3d_b200 import weights as Wt
from hand3d_b200.frames import FrameRunner, to_network_input

pytestmark = pytest.mark.gpu
F = np.float32
W_SEG = Wt.synthetic_weights(0, seg_shift=0.15)   # blob images give varied masks with these


@pytest.fixture(scope="module")
def ctx():
    c = runtime.Context()
    c.load_weights(W_SEG)
    yield c
    torch.cuda.synchronize()
    c.release_graphs()


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _hands(rng, B, H, W):
    """B hand-shaped skeletons about a third of the frame high, some reaching off the image, with non-finite joints in some."""
    size = np.float32([H, W]) / 3
    base = rng.uniform(-0.1, 0.9, (B, 1, 2)).astype(F) * np.float32([H, W])
    c = (base + rng.uniform(0, 1, (B, 21, 2)).astype(F) * size).astype(F)
    if B > 1:
        c[1, 3, 0] = np.nan
        c[1, 7, 1] = np.inf
    if B > 2:
        c[2] = -c[2] - 100.0            # wholly off the image
    return c


def _spans(rng, B, H, W, S=24):
    seg = (rng.uniform(-0.2, 1.2, (B, S, 4)) * np.float32([H, W, H, W])).astype(F)
    if B > 1:
        seg[1, 5, 2] = -np.inf
        seg[1, 6, 0] = np.nan
        seg[1, 7] = [1e30, -1e30, -1e30, 1e30]
    return seg


def _case(B, H, W, kind, seed):
    rng = np.random.default_rng(seed)
    imgs = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
    if kind == "hand":
        seg, cols = O.hand_segments(_hands(rng, B, H, W), D.BONES), D.PALETTE
    else:
        seg, cols = _spans(rng, B, H, W), rng.uniform(0, 255, (24, 3)).astype(F)
    valid = (rng.uniform(size=B) < 0.75).astype(np.int32) if B > 1 else None
    return imgs, seg, cols, valid


def _draw_dev(ctx, imgs, seg, cols, lw, valid):
    t = _dev(imgs)
    ctx.draw_segments(t, _dev(seg), cols, lw, None if valid is None else _dev(valid))
    return t.cpu().numpy()


SIZES = [(1, 240, 320), (3, 240, 320), (32, 240, 320), (1, 1080, 1920), (3, 1080, 1920), (32, 1080, 1920), (1, 2160, 3840),
         (2, 2160, 3840), (1, 4096, 4096)]


@pytest.mark.parametrize("lw", [0.5, 1.0, 4.5, 64.0])
@pytest.mark.parametrize("B,H,W", SIZES)
def test_hands_equal_oracle(ctx, B, H, W, lw):
    imgs, seg, cols, valid = _case(B, H, W, "hand", B * 7 + H)
    np.testing.assert_array_equal(_draw_dev(ctx, imgs, seg, cols, lw, valid), O.draw(imgs, seg, cols, lw, valid))


@pytest.mark.parametrize("lw", [0.5, 1.0, 4.5, 64.0])
@pytest.mark.parametrize("B,H,W", [(1, 240, 320), (3, 240, 320), (1, 1080, 1920), (3, 1080, 1920)])
def test_frame_spanning_segments_equal_oracle(ctx, B, H, W, lw):
    imgs, seg, cols, valid = _case(B, H, W, "span", B * 11 + W)
    np.testing.assert_array_equal(_draw_dev(ctx, imgs, seg, cols, lw, valid), O.draw(imgs, seg, cols, lw, valid))


def test_huge_end_points_follow_the_box(ctx):
    """End points far beyond 2^14 px, where the rule's per-segment box decides what a long segment reaches."""
    rng = np.random.default_rng(9)
    imgs = rng.integers(0, 256, (2, 240, 320, 3), dtype=np.uint8)
    seg = np.float32([[[10.0, -1e8, 10.0, 101.0], [-3e7, 50.0, 200.0, 50.0], [100.0, 5e8, 120.0, 200.0], [1e9, 1e9, 5.0, 5.0]],
                      [[120.0, -2e9, 121.5, 319.0], [-4e6, -4e6, 239.0, 319.0], [60.0, 60.0, 6e7, 6e7], [0.0, 160.0, 2e8, 160.0]]])
    cols = rng.uniform(0, 255, (4, 3)).astype(F)
    for lw in (1.0, 4.5):
        np.testing.assert_array_equal(_draw_dev(ctx, imgs, seg, cols, lw, None), O.draw(imgs, seg, cols, lw))


@pytest.mark.parametrize("H,W", [(1, 1), (1, 700), (700, 1), (7, 5)])
def test_tiny_images(ctx, H, W):
    rng = np.random.default_rng(H * W)
    imgs = rng.integers(0, 256, (2, H, W, 3), dtype=np.uint8)
    seg = (rng.uniform(-1, 1.5, (2, 6, 4)) * np.float32([H, W, H, W])).astype(F)
    cols = rng.uniform(0, 255, (6, 3)).astype(F)
    for lw in (0.5, 3.0):
        np.testing.assert_array_equal(_draw_dev(ctx, imgs, seg, cols, lw, None), O.draw(imgs, seg, cols, lw))


def test_draw_hand_equals_draw_segments(ctx):
    rng = np.random.default_rng(5)
    B, H, W = 4, 240, 320
    imgs = rng.integers(0, 256, (B, H, W, 3), dtype=np.uint8)
    hw = _hands(rng, B, H, W).astype(np.float64) + 0.123456789
    seg = O.hand_segments(hw, D.BONES)
    want = _draw_dev(ctx, imgs, seg, D.PALETTE, 2.0, None)
    np.testing.assert_array_equal(D.draw_hand(_dev(imgs), hw, linewidth=2.0).cpu().numpy(), want)          # numpy float64
    np.testing.assert_array_equal(D.draw_hand(_dev(imgs), _dev(hw), linewidth=2.0).cpu().numpy(), want)    # CUDA float64
    one = D.draw_hand(_dev(imgs[1]), _dev(hw[1].astype(F)), linewidth=2.0)                                  # [H,W,3]
    np.testing.assert_array_equal(one.cpu().numpy(), want[1])
    fixed = np.repeat(np.float32(255.0 * np.array([0.25, 0.5, 0.75]))[None], 20, 0)
    valid = np.int32([1, 0, 1, 1])
    np.testing.assert_array_equal(D.draw_hand(_dev(imgs), hw, color_fixed=(0.25, 0.5, 0.75), valid=_dev(valid)).cpu().numpy(),
                                  O.draw(imgs, seg, fixed, 1.0, valid))


def test_draw_hand_3d_equals_oracle(ctx):
    rng = np.random.default_rng(6)
    xyz = rng.normal(scale=1.2, size=(3, 21, 3)).astype(F)
    panels = np.full((3,) + D.PANEL_3D + (3,), 255, np.uint8)
    got = D.draw_hand_3d(_dev(panels), _dev(xyz)).cpu().numpy()
    hw = O.project_3d(xyz, *D.PANEL_3D)
    np.testing.assert_array_equal(D.project_3d(_dev(xyz), D.PANEL_3D).cpu().numpy(), hw)
    np.testing.assert_array_equal(got, O.draw(panels, O.hand_segments(hw, D.BONES), D.PALETTE, 1.0))
    assert (got != 255).any()


def test_run_figure_panels(ctx):
    ctx.set_precision("bf16x3")
    frames = np.clip(np.round((Wt.synthetic_blob_images(2, 240, 320, seed=21) + 0.5) * 255.0), 0, 255).astype(np.uint8)
    image_u8 = _dev(frames)
    r = ctx.pipeline(to_network_input(image_u8), _dev(np.float32([[1.0, 0.0]] * 2)), True, outputs="all")
    fig = D.run_figure(image_u8, r)
    crop = r["image_crop"].cpu().numpy()
    want_crop = np.clip((crop + F(0.5)) * F(255), 0, 255).astype(np.uint8)
    uv = r["keypoints_uv"].cpu().numpy()
    np.testing.assert_array_equal(fig["crop"].cpu().numpy(), O.draw(want_crop, O.hand_segments(uv, D.BONES), D.PALETTE, 1.0))
    hs = r["hand_scoremap"].cpu().numpy()
    np.testing.assert_array_equal(fig["mask"].cpu().numpy(), D.VIRIDIS_ENDS[np.argmax(hs, 3)])
    kp = D.trafo_coords(uv.astype(np.float64), r["center"].cpu().numpy()[:, None], r["scale_crop"].cpu().numpy()[:, None], 256)
    np.testing.assert_array_equal(fig["image"].cpu().numpy(), O.draw(frames, O.hand_segments(kp, D.BONES), D.PALETTE, 1.0))
    np.testing.assert_array_equal(image_u8.cpu().numpy(), frames)          # the input is not drawn on
    assert tuple(fig["grid"].shape) == (2, 512, 720, 3) and tuple(fig["pose3d"].shape) == (2,) + D.PANEL_3D + (3,)


def test_poisoned_scratch_gives_the_same_bits(ctx):
    imgs, seg, cols, valid = _case(3, 1080, 1920, "hand", 77)
    out = []
    for byte in (0, 0xFF):
        ctx.fill_scratch(byte)
        out.append(_draw_dev(ctx, imgs, seg, cols, 4.5, valid))
    np.testing.assert_array_equal(out[0], out[1])


def test_captured_draw_replays_equal_to_eager(ctx):
    imgs, seg, cols, valid = _case(3, 1080, 1920, "span", 78)
    t, s, v = _dev(imgs), _dev(seg), _dev(valid)
    eager = t.clone()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ctx.draw_segments(t, s, cols, 3.0, v)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(t.cpu().numpy(), imgs)              # capturing enqueued nothing
    torch.cuda.set_sync_debug_mode("error")
    try:
        ctx.draw_segments(eager, s, cols, 3.0, v)
        ctx.draw_segments(eager, s, cols, 3.0, v)
        g.replay()
        g.replay()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    np.testing.assert_array_equal(t.cpu().numpy(), eager.cpu().numpy())


def test_bad_arguments_are_refused_before_any_launch(ctx):
    B, H, W, S = 2, 64, 64, 3
    img = torch.zeros((B, H, W, 3), dtype=torch.uint8, device="cuda")
    seg = torch.zeros((B, S, 4), dtype=torch.float32, device="cuda")
    good = np.full((S, 3), 100.0, F)
    P = C.c_void_p

    def call(images=img, b=B, h=H, w=W, segments=seg, s=S, colors=good, lw=1.0):
        cp = None if colors is None else np.ascontiguousarray(colors, F).ctypes.data_as(P)
        return ctx.lib.h3d_draw_segments(ctx.h, None if images is None else P(images.data_ptr()), b, h, w,
                                         None if segments is None else P(segments.data_ptr()), s, cp, None, C.c_float(lw),
                                         P(torch.cuda.current_stream().cuda_stream))
    assert call() == _lib.OK
    torch.cuda.synchronize()
    n0 = ctx.launch_count
    nan, inf = float("nan"), float("inf")
    bad_cols = [np.full((S, 3), -1.0, F), np.full((S, 3), 255.5, F), np.full((S, 3), nan, F), np.full((S, 3), inf, F)]
    cases = [dict(images=None), dict(segments=None), dict(colors=None), dict(b=0), dict(h=0), dict(w=0), dict(h=4097),
             dict(w=4097), dict(s=0), dict(s=65), dict(lw=0.0), dict(lw=-1.0), dict(lw=64.5), dict(lw=nan), dict(lw=inf)]
    cases += [dict(colors=c) for c in bad_cols]
    for case in cases:
        assert call(**case) == _lib.EINVAL, case
        assert ctx.launch_count == n0, case
    assert b"h3d_draw_segments" in ctx.lib.h3d_last_error()
    assert call(lw=64.0) == _lib.OK and ctx.launch_count == n0 + 1
    with pytest.raises(ValueError):
        ctx.draw_segments(img, seg, np.zeros((S + 1, 3), F))
    with pytest.raises(RuntimeError):
        ctx.draw_segments(img, seg, np.full((S, 3), 300.0, F))


# ------------------------------------------------------------------------------------------- FrameRunner(draw=True)
FRAME_HW = (1080, 1920)
BATCH = 8
COLORS = np.concatenate([np.repeat(D.WHITE[None], 4, 0), D.PALETTE])


def _uint8(img):
    return np.clip(np.round((img + 0.5) * 255.0), 0, 255).astype(np.uint8)


def _sequence(n, noise_at):
    """BATCH streams of a blob frame shifted (2, 3) px per step; stream 0 gets a faint-noise frame at noise_at."""
    base = _uint8(Wt.synthetic_blob_images(BATCH, FRAME_HW[0], FRAME_HW[1], seed=21))
    rng = np.random.default_rng(22)
    frames = []
    for t in range(n):
        f = np.stack([np.roll(base[b], (2 * t, 3 * t), axis=(0, 1)) for b in range(BATCH)])
        if t == noise_at:
            f[0] = rng.integers(126, 131, f[0].shape, dtype=np.uint8)
        frames.append(f)
    return frames


def _want_drawn(frames, res, lost=None, size=(240, 320)):
    seg = np.concatenate([O.crop_box(res["center"], res["scale_crop"], FRAME_HW, size),
                          O.hand_segments(res["keypoints_frame"].astype(F), D.BONES)], 1)
    valid = None if lost is None else (~np.asarray(lost, bool)).astype(np.int32)
    return O.draw(frames, seg, COLORS, 4.5, valid)


def _check(frames, plain, drawn, lost_key=None, size=(240, 320), drawn_every=1):
    assert len(plain) == len(drawn) == len(frames)
    for t, (p, q, f) in enumerate(zip(plain, drawn, frames)):
        read = drawn_every > 0 and t % drawn_every == 0
        assert set(q) == set(p) | ({"frame_drawn"} if read else set()), (t, set(q), set(p))
        for k in p:
            np.testing.assert_array_equal(np.asarray(q[k]), np.asarray(p[k]), err_msg="%s at step %d" % (k, t))
        if not read:
            continue
        lost = None if lost_key is None else q[lost_key]
        np.testing.assert_array_equal(q["frame_drawn"], _want_drawn(f, q, lost, size), err_msg="frame_drawn at step %d" % t)
        if lost is not None:
            for b in np.flatnonzero(lost):
                np.testing.assert_array_equal(q["frame_drawn"][b], f[b])


def _submit_all(runner, frames):
    out = []
    for f in frames:
        r = runner.submit(_dev(f))
        out.append({k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in r.items()})
    return out


def test_frame_runner_draw_submit_and_stream(ctx):
    ctx.set_precision("bf16x3")
    frames = _sequence(3, noise_at=None)
    try:
        plain = FrameRunner(ctx, BATCH, FRAME_HW)
        drawn = FrameRunner(ctx, BATCH, FRAME_HW, draw=True)
        assert drawn.draw_linewidth == 4.5
        _check(frames, _submit_all(plain, frames), _submit_all(drawn, frames))
        _check(frames, list(plain.stream(frames)), list(drawn.stream(frames)))
    finally:
        ctx.release_graphs()


def test_frame_runner_draw_at_another_network_size(ctx):
    """size=(320, 320): the crop square is mapped to the frame from the network image the step used, as the key-points are; and
    stream(drawn_every=2) reads the drawn frames of batches 0 and 2 only."""
    ctx.set_precision("bf16x3")
    size = (320, 320)
    frames = _sequence(3, noise_at=None)
    try:
        plain = FrameRunner(ctx, BATCH, FRAME_HW, size=size)
        drawn = FrameRunner(ctx, BATCH, FRAME_HW, size=size, draw=True)
        sub = _submit_all(drawn, frames)
        _check(frames, _submit_all(plain, frames), sub, size=size)
        _check(frames, list(plain.stream(frames)), list(drawn.stream(frames, drawn_every=2)), size=size, drawn_every=2)
        none = list(drawn.stream(frames, drawn_every=0))
        assert all("frame_drawn" not in r for r in none)
        with pytest.raises(ValueError):
            list(drawn.stream(frames, drawn_every=-1))
    finally:
        ctx.release_graphs()
    # the square FrameRunner draws: crop_box_segments with the runner's size equals the oracle's at that size, which is not the
    # 240x320 mapping (the squares of these steps may lie partly off the frames, so the bytes alone need not tell the two apart)
    r = sub[0]
    got = D.crop_box_segments(_dev(r["center"]), _dev(r["scale_crop"]), FRAME_HW, size).cpu().numpy()
    np.testing.assert_array_equal(got, O.crop_box(r["center"], r["scale_crop"], FRAME_HW, size))
    assert (got != O.crop_box(r["center"], r["scale_crop"], FRAME_HW)).any()


@pytest.mark.parametrize("detect", ["batch", "slots"])
def test_frame_runner_draw_skips_lost_slots(ctx, detect):
    ctx.set_precision("bf16x3")
    n, noise_at = 6, 3
    frames = _sequence(n, noise_at)
    kw = dict(track=True, detect=detect, track_margin=1.5)
    try:
        free = list(FrameRunner(ctx, BATCH, FRAME_HW, **kw).stream(frames))
        sc = np.array([r["track_score"] for r in free])
        others = np.delete(sc.reshape(-1), noise_at * BATCH)
        lo = sc[noise_at, 0]
        min_score = float((lo + others.min()) / 2) if lo < others.min() else float(np.nextafter(F(lo), F(np.inf)))
        plain = FrameRunner(ctx, BATCH, FRAME_HW, min_score=min_score, **kw)
        drawn = FrameRunner(ctx, BATCH, FRAME_HW, min_score=min_score, draw=True, **kw)
        p_stream, d_stream = list(plain.stream(frames)), list(drawn.stream(frames))
        _check(frames, p_stream, d_stream, "track_lost")
        plain = FrameRunner(ctx, BATCH, FRAME_HW, min_score=min_score, **kw)
        drawn = FrameRunner(ctx, BATCH, FRAME_HW, min_score=min_score, draw=True, **kw)
        p_sub, d_sub = _submit_all(plain, frames), _submit_all(drawn, frames)
        _check(frames, p_sub, d_sub, "track_lost")
    finally:
        ctx.release_graphs()
    lost = np.array([r["track_lost"] for r in d_stream])
    assert lost[noise_at, 0] and not lost.all(), lost

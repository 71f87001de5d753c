"""Camera rigs on the device (h3d_resize_frames_rig, FrameRunner with per-slot sizes and formats): every slot equals, bit for bit, the
single-camera path fed that slot's frame alone (to_network_input, a one-camera FrameRunner, Context.track_step / track_step_slots
on the stacked per-slot network images), and tests/frames_yuv_oracle.py cross-checks small sizes on the CPU."""
import os

import numpy as np
import pytest
import torch

import frames_oracle as F
import frames_yuv_oracle as Y
from hand3d_b200 import _lib, runtime
from hand3d_b200 import frames as FR
from hand3d_b200 import weights as Wt
from hand3d_b200.utils.general import trafo_coords

pytestmark = pytest.mark.gpu

# 2..8 slots, at least three sizes each (one not a multiple of 8, one above 2048 px), all five formats
RIGS = {
    "3cams": (["nv12", "rgb", "yuyv"], [(1080, 1920), (722, 1282), (480, 640)]),
    "5fmts": (["i420", "bgr", "nv12", "yuyv", "rgb"], [(2160, 3840), (243, 321), (720, 1280), (100, 78), (1080, 1920)]),
    "8cams": (["rgb", "i420", "i420", "yuyv", "bgr", "nv12", "yuyv", "rgb"],
              [(2, 2050), (720, 1280), (720, 1280), (481, 642), (4096, 4096), (2, 2), (1080, 1920), (1, 1)]),
    "2cams": (["bgr", "nv12"], [(2304, 4096), (362, 498)]),
}
RUNNER_RIG = (["nv12", "rgb", "yuyv", "i420"], [(1080, 1920), (722, 1282), (480, 640), (720, 1280)])


@pytest.fixture(scope="module")
def ctx():
    c = runtime.Context()
    c.load_weights(Wt.synthetic_weights(0))
    yield c
    c.release_graphs()


def _frames(fmts, hws, seed):
    return [Y.random_frame(seed + 7 * b, f, *hw) for b, (f, hw) in enumerate(zip(fmts, hws))]


def _blob_frames(fmts, hws, t, seed=21, noise=None):
    """Step t of a moving blob per camera, scaled (nearest) to each camera's size and packed into its format; noise: a faint-noise
    frame for that slot instead."""
    B = len(fmts)
    base = np.clip(np.round((Wt.synthetic_blob_images(B, 240, 320, seed=seed) + 0.5) * 255.0), 0, 255).astype(np.uint8)
    out = []
    for b, (f, (H, W)) in enumerate(zip(fmts, hws)):
        img = np.roll(base[b], (2 * t, 3 * t), axis=(0, 1))
        if noise == b:
            img = np.random.default_rng(22 + t).integers(126, 131, img.shape, dtype=np.uint8)
        rgb = img[(np.arange(H) * 240 // H)[:, None], (np.arange(W) * 320 // W)[None, :]]
        if f == "rgb":
            out.append(np.ascontiguousarray(rgb))
        elif f == "bgr":
            out.append(np.ascontiguousarray(rgb[..., ::-1]))
        else:
            Yp = np.clip(16 + (rgb.astype(np.int32) @ np.array([66, 129, 25])) // 256, 0, 255).astype(np.uint8)
            ch = (H // 2, W // 2) if f in ("nv12", "i420") else (H, W // 2)
            U = np.full(ch, 110, np.uint8)
            V = np.full(ch, 150, np.uint8)
            out.append(Y.pack(f, Yp, U, V))
    return out


def _host(r):
    return {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else [x.cpu().numpy() for x in v] if isinstance(v, list) else v)
            for k, v in r.items()}


def _bits(a, b, msg):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, (msg, a.shape, b.shape, a.dtype, b.dtype)
    np.testing.assert_array_equal(a.view(np.uint8), b.view(np.uint8), err_msg=msg)


# ------------------------------------------------------------------------------------------------------------------ the resize
@pytest.mark.parametrize("rig", list(RIGS))
@pytest.mark.parametrize("out_hw", [(240, 320), (256, 256)], ids=lambda s: "%dx%d" % s)
def test_rig_resize_equals_each_frame_alone(ctx, rig, out_hw):
    fmts, hws = RIGS[rig]
    frames = [torch.from_numpy(f).cuda() for f in _frames(fmts, hws, seed=len(rig) + out_hw[1])]
    for normalize in (False, True):
        got = ctx.resize_frames_rig(frames, *out_hw, normalize=normalize, pixel_formats=fmts)
        for b, (fr, f) in enumerate(zip(frames, fmts)):
            want = ctx.resize_frames(fr.unsqueeze(0), *out_hw, normalize=normalize, pixel_format=f)[0]
            _bits(got[b].cpu().numpy(), want.cpu().numpy(), "slot %d (%s %s), normalize=%d" % (b, f, hws[b], normalize))
            if normalize and out_hw == FR.NETWORK_SIZE:
                alone = FR.to_network_input(fr, pixel_format=f)
                _bits(got[b].cpu().numpy(), alone.cpu().numpy(), "slot %d against to_network_input" % b)
    # the CPU restatement on the small slots
    host = ctx.resize_frames_rig(frames, *out_hw, normalize=False, pixel_formats=fmts).cpu().numpy()
    for b, (fr, f, hw) in enumerate(zip(frames, fmts, hws)):
        if hw[0] * hw[1] <= 800 * 800:
            np.testing.assert_array_equal(host[b], Y.resize(f, fr.cpu().numpy(), *out_hw), err_msg="slot %d restated" % b)


def test_rig_resize_launches_one_kernel_per_format_and_is_capturable(ctx):
    fmts, hws = RIGS["8cams"]
    frames = [torch.from_numpy(f).cuda() for f in _frames(fmts, hws, seed=5)]
    out = torch.empty((8, 240, 320, 3), dtype=torch.float32, device="cuda")
    ctx.resize_frames_rig(frames, 240, 320, True, out=out, pixel_formats=fmts)   # builds the plan
    torch.cuda.synchronize()
    n0 = ctx.launch_count
    ctx.resize_frames_rig(frames, 240, 320, True, out=out, pixel_formats=fmts)
    assert ctx.launch_count - n0 == len(set(fmts)) == 5
    want = out.clone()
    out.zero_()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ctx.resize_frames_rig(frames, 240, 320, True, out=out, pixel_formats=fmts)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    del g
    # a rig without a plan is refused under capture, before anything is enqueued
    other = [torch.zeros(Y.frame_shape(f, *hw), dtype=torch.uint8, device="cuda") for f, hw in zip(["rgb", "yuyv"], [(30, 40), (32, 44)])]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with pytest.raises(RuntimeError, match="no plan"):
            with torch.cuda.graph(g, stream=s):
                ctx.resize_frames_rig(other, 240, 320, True, pixel_formats=["rgb", "yuyv"])
    torch.cuda.synchronize()


def test_rig_resize_refusals(ctx):
    good = [torch.zeros((8, 8, 3), dtype=torch.uint8, device="cuda"), torch.zeros((12, 8), dtype=torch.uint8, device="cuda")]
    n0 = ctx.launch_count
    with pytest.raises(ValueError, match="slot 1"):
        ctx.resize_frames_rig([good[0], torch.zeros((13, 8), dtype=torch.uint8, device="cuda")], 240, 320, True, pixel_formats=["rgb", "nv12"])
    with pytest.raises(TypeError, match="slot 0"):
        ctx.resize_frames_rig([good[0].float(), good[1]], 240, 320, True, pixel_formats=["rgb", "nv12"])
    with pytest.raises(ValueError, match="pixel formats"):
        ctx.resize_frames_rig(good, 240, 320, True, pixel_formats=["rgb"])
    with pytest.raises(ValueError, match="slot 1"):
        ctx.resize_frames_rig(good, 240, 320, True, pixel_formats=["rgb", "rgba"])
    with pytest.raises(ValueError, match="one frame per slot"):
        ctx.resize_frames_rig([good[0].expand(2, 8, 8, 3).contiguous(), good[1]], 240, 320, True, pixel_formats=["rgb", "nv12"])
    with pytest.raises(RuntimeError, match="slot 1"):       # odd 4:2:0 width, refused by the library
        ctx.resize_frames_rig([good[0], torch.zeros((12, 7), dtype=torch.uint8, device="cuda")], 240, 320, True, pixel_formats=["rgb", "nv12"])
    with pytest.raises(RuntimeError, match="slot 0"):
        ctx.resize_frames_rig([torch.zeros((4097, 1, 3), dtype=torch.uint8, device="cuda"), good[1]], 240, 320, True,
                              pixel_formats=["rgb", "nv12"])
    torch.cuda.synchronize()
    assert ctx.launch_count == n0


def test_rig_resize_on_poisoned_workspace_and_scratch(ctx):
    fmts, hws = RIGS["5fmts"]
    frames = [torch.from_numpy(f).cuda() for f in _frames(fmts, hws, seed=90)]
    ctx.ensure_workspace(5, 240, 320)

    def run():
        return [ctx.resize_frames_rig(frames, 240, 320, normalize=n, pixel_formats=fmts).cpu() for n in (False, True)]
    clean = run()
    for byte in (0x00, 0xFF, 0x7F):
        ctx.fill_scratch(byte)
        for a, b in zip(run(), clean):
            assert torch.equal(a, b), "a result changed after a 0x%02X fill" % byte
    ctx.check_errors()


# ------------------------------------------------------------------------------------------------------------------ frame_coords
def test_frame_coords_per_slot_equals_per_size(ctx):
    rng = np.random.default_rng(3)
    c = torch.from_numpy(rng.uniform(-20, 260, (4, 21, 2))).cuda()
    hws = RUNNER_RIG[1]
    got = FR.frame_coords(c, torch.tensor(hws, dtype=torch.float64, device="cuda"))
    got_list = FR.frame_coords(c, hws)
    for b, hw in enumerate(hws):
        want = FR.frame_coords(c[b:b + 1], hw)
        _bits(got[b:b + 1].cpu().numpy(), want.cpu().numpy(), "slot %d" % b)
        _bits(got_list[b:b + 1].cpu().numpy(), want.cpu().numpy(), "slot %d from a list" % b)
        np.testing.assert_array_equal(got[b].cpu().numpy(), F.frame_coords(c[b].cpu().numpy(), hw))


# ------------------------------------------------------------------------------------------------------------------ FrameRunner
def _one_camera_runs(ctx, fmts, hws, steps, **kw):
    """Each camera through its own one-camera FrameRunner: per step, per slot, its host results."""
    per_slot = []
    for b, (f, hw) in enumerate(zip(fmts, hws)):
        r1 = FR.FrameRunner(ctx, 1, hw, pixel_format=f, **kw)
        per_slot.append([_host(r1.submit(s[b][None])) for s in steps])
        del r1
        ctx.release_graphs()
    return per_slot


def test_runner_equals_one_camera_runners_and_draws_each_camera(ctx):
    fmts, hws = RUNNER_RIG
    steps = [_blob_frames(fmts, hws, t) for t in range(3)]
    runner = FR.FrameRunner(ctx, 4, hws, draw=True, pixel_format=fmts)
    assert runner.rig and runner.frame_hw == hws and runner.pixel_format == fmts
    got = []
    for t, s in enumerate(steps):                  # host, CUDA and mixed submissions
        sub = s if t == 0 else [torch.from_numpy(x).cuda() for x in s] if t == 1 else [x if b % 2 else torch.from_numpy(x).cuda()[None]
                                                                                         for b, x in enumerate(s)]
        got.append(_host(runner.submit(sub)))
    del runner
    ctx.release_graphs()
    want = _one_camera_runs(ctx, fmts, hws, steps, draw=True)
    for t in range(len(steps)):
        assert isinstance(got[t]["frame_drawn"], list) and len(got[t]["frame_drawn"]) == 4
        for b in range(4):
            w = want[b][t]
            for k in FR.FrameRunner.RESULT_KEYS:
                _bits(got[t][k][b:b + 1], w[k], "%s of slot %d at step %d" % (k, b, t))
            assert got[t]["frame_drawn"][b].shape == hws[b] + (3,)
            _bits(got[t]["frame_drawn"][b], w["frame_drawn"][0], "frame_drawn of slot %d at step %d" % (b, t))
    # the key-points drawn are the ones reported, in each slot's own frame pixels
    r = got[0]
    kp = FR.frame_coords(trafo_coords(torch.from_numpy(r["keypoints_uv"]).cuda(), torch.from_numpy(r["center"]).cuda(),
                                      torch.from_numpy(r["scale_crop"]).cuda(), 256), hws)
    _bits(kp.cpu().numpy(), r["keypoints_frame"], "keypoints_frame")


def test_runner_stream_equals_submit_and_host_equals_cuda(ctx):
    fmts, hws = RUNNER_RIG
    steps = [_blob_frames(fmts, hws, t, seed=31) for t in range(4)]
    hs = np.array([[0.0, 1.0], [1.0, 0.0], [0.0, 1.0], [1.0, 0.0]], np.float32)
    runner = FR.FrameRunner(ctx, 4, hws, draw=True, pixel_format=fmts, track=True, detect="slots")
    streamed = list(runner.stream([(s, hs) if t % 2 else s for t, s in enumerate(steps)], drawn_every=2))
    del runner
    ctx.release_graphs()
    for dev in (False, True):
        runner = FR.FrameRunner(ctx, 4, hws, draw=True, pixel_format=fmts, track=True, detect="slots")
        for t, s in enumerate(steps):
            r = _host(runner.submit([torch.from_numpy(x).cuda() for x in s] if dev else s, hs if t % 2 else None))
            for k, v in streamed[t].items():
                if k == "frame_drawn":
                    assert t % 2 == 0
                    for b in range(4):
                        _bits(v[b], r[k][b], "frame_drawn %d at step %d" % (b, t))
                else:
                    _bits(v, r[k], "%s at step %d (cuda=%d)" % (k, t, dev))
            assert ("frame_drawn" in streamed[t]) == (t % 2 == 0)
        del runner
        ctx.release_graphs()


@pytest.mark.parametrize("detect", ["batch", "slots"])
def test_runner_tracking_equals_track_step_on_network_images(ctx, detect):
    ctx.set_precision("bf16x3")
    fmts, hws = RUNNER_RIG
    n, noise_at = 7, 3
    steps = [_blob_frames(fmts, hws, t, noise=0 if t == noise_at else None) for t in range(n)]
    kw = dict(track=True, detect=detect, redetect_every=None)
    try:
        free = list(FR.FrameRunner(ctx, 4, hws, pixel_format=fmts, **kw).stream(steps))
        min_score = float(np.nextafter(np.float32(free[noise_at]["track_score"][0]), np.float32(np.inf)))
        res = list(FR.FrameRunner(ctx, 4, hws, pixel_format=fmts, min_score=min_score, **kw).stream(steps))
    finally:
        ctx.release_graphs()
    assert res[noise_at]["track_lost"][0], "slot 0 is meant to be lost at the noise step"
    st = runtime.TrackState(4)
    hs = torch.tensor([[1.0, 0.0]] * 4, dtype=torch.float32, device="cuda")
    for t, s in enumerate(steps):
        image = torch.cat([FR.to_network_input(torch.from_numpy(x).cuda(), pixel_format=f)[None] for x, f in zip(s, fmts)])
        if detect == "slots":
            r = ctx.track_step_slots(image, hs, st, margin=1.5, min_score=min_score, outputs="keypoints")
        else:
            r = ctx.track_step(image, hs, st, res[t]["detected"], margin=1.5, min_score=min_score, outputs="keypoints")
        r["keypoints_frame"] = FR.frame_coords(trafo_coords(r["keypoints_uv"], r["center"], r["scale_crop"], 256), hws)
        r["track_score"] = st.score.clone()
        r["track_lost"] = st.lost != 0
        r = _host(r)
        for k in res[t]:
            if k != "detected":
                _bits(res[t][k], r[k], "%s at step %d" % (k, t))
    if detect == "batch":
        assert res[noise_at + 2]["detected"]      # a slot lost at t makes step t + 2 a detect step


def test_lost_slots_are_not_drawn(ctx):
    ctx.set_precision("bf16x3")
    fmts, hws = RUNNER_RIG
    steps = [_blob_frames(fmts, hws, t, noise=1 if t == 1 else None) for t in range(3)]
    free = list(FR.FrameRunner(ctx, 4, hws, pixel_format=fmts, track=True, detect="slots").stream(steps))
    ctx.release_graphs()
    min_score = float(np.nextafter(np.float32(free[1]["track_score"][1]), np.float32(np.inf)))
    res = list(FR.FrameRunner(ctx, 4, hws, pixel_format=fmts, track=True, detect="slots", min_score=min_score, draw=True).stream(steps))
    ctx.release_graphs()
    lost = res[1]["track_lost"]
    assert lost[1]
    for b in range(4):
        rgb = Y.to_rgb(fmts[b], steps[1][b])
        assert np.array_equal(res[1]["frame_drawn"][b], rgb) == bool(lost[b]), "slot %d (lost=%d)" % (b, lost[b])


def test_all_equal_rig_takes_the_single_size_path(ctx):
    hw, fmt = (480, 640), "nv12"
    per_cam = [_blob_frames([fmt] * 3, [hw] * 3, t) for t in range(3)]
    steps = [np.stack(c) for c in per_cam]
    runs = []
    for frame_hw, pf in ((hw, fmt), ([hw] * 3, [fmt] * 3), ([hw] * 3, fmt), (hw, [fmt] * 3)):
        runner = FR.FrameRunner(ctx, 3, frame_hw, draw=True, pixel_format=pf)
        assert not runner.rig and runner.frame_hw == hw and runner.pixel_format == fmt
        assert runner._frames[0].shape == (3,) + Y.frame_shape(fmt, *hw)
        listed = isinstance(frame_hw, list) or isinstance(pf, list)
        assert runner.per_slot == listed
        assert runner.draw_linewidth == ([2.0] * 3 if listed else 2.0)
        out = []
        for t, s in enumerate(steps):               # a stacked batch, a list of host frames, a mixed list of host and CUDA frames
            sub = s if t == 0 else per_cam[t] if t == 1 else [x if b == 1 else torch.from_numpy(x).cuda() for b, x in enumerate(per_cam[t])]
            r = _host(runner.submit(sub))
            if listed:                                # a rig's frame_drawn: one [H,W,3] image per slot
                assert isinstance(r["frame_drawn"], list) and len(r["frame_drawn"]) == 3
                r["frame_drawn"] = np.stack(r["frame_drawn"])
            out.append(r)
        if listed:
            streamed = list(runner.stream([per_cam[0], (per_cam[1], None)]))
            for t in range(2):
                assert isinstance(streamed[t]["frame_drawn"], list)
                _bits(np.stack(streamed[t]["frame_drawn"]), out[t]["frame_drawn"], "streamed frame_drawn at step %d" % t)
        runs.append(out)
        del runner
        ctx.release_graphs()
    for run in runs[1:]:
        for t in range(len(steps)):
            for k in runs[0][t]:
                _bits(run[t][k], runs[0][t][k], "%s at step %d" % (k, t))


def test_mixed_submission_reads_cuda_frames_in_stream_order(ctx):
    """A CUDA frame still being written on the current stream when submit() is called is read after it is complete, and may be
    freed right after submit()."""
    fmts, hws = RUNNER_RIG
    steps = [_blob_frames(fmts, hws, t, seed=51) for t in range(2)]
    runner = FR.FrameRunner(ctx, 4, hws, pixel_format=fmts, draw=True)
    want = [_host(runner.submit([torch.from_numpy(x).cuda() for x in s])) for s in steps]
    got = []
    for s in steps:
        src = [torch.from_numpy(x).cuda() for x in s]
        torch.cuda.synchronize()
        late = [torch.zeros_like(x) for x in src]
        torch.cuda._sleep(20_000_000)               # the current stream is busy, then writes the CUDA frames
        for d, x in zip(late, src):
            d.copy_(x)
        r = runner.submit([late[0], s[1], late[2], s[3]])
        del late, src                               # freed while the copies may still be pending
        got.append(_host(r))
    for t in range(len(steps)):
        for k in want[t]:
            if k == "frame_drawn":
                for b in range(4):
                    _bits(got[t][k][b], want[t][k][b], "frame_drawn %d at step %d" % (b, t))
            else:
                _bits(got[t][k], want[t][k], "%s at step %d" % (k, t))
    del runner
    ctx.release_graphs()


def _demo(tmp_path, *args):
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "examples", "run_frames_demo.py"), *args], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=900, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout[-4000:]
    return r.stdout


@pytest.mark.parametrize("sources", [["synthetic:nv12:1080x1920", "synthetic:yuyv:722x1282", "synthetic:bgr:481x642"],
                                     ["synthetic:nv12:480x640"], ["synthetic:i420:480x640"] * 2], ids=["mixed", "one", "equal"])
def test_demo_with_sources(tmp_path, sources):
    from PIL import Image
    args = [a for s in sources for a in ("--source", s)]
    out = _demo(tmp_path, *args, "--batches", "3", "--track", "--detect", "slots", "--draw-dir", str(tmp_path / "drawn"))
    assert out.count("batch ") >= 3 and "frames/s" in out
    for b, s in enumerate(sources):
        H, W = (int(v) for v in s.rsplit(":", 1)[1].split("x"))
        im = Image.open(tmp_path / "drawn" / ("batch000_frame%02d.png" % b))
        assert im.size == (W, H) and im.mode == "RGB"
    assert len(os.listdir(tmp_path / "drawn")) == len(sources)


def test_demo_with_todays_flags(tmp_path):
    out = _demo(tmp_path, "--batch", "2", "--batches", "2", "--height", "480", "--width", "640", "--track", "--draw-dir",
                str(tmp_path / "drawn"))
    assert out.count("batch ") >= 2 and "in 480x640 pixels" in out
    assert len(os.listdir(tmp_path / "drawn")) == 2


def test_runner_refusals(ctx):
    fmts, hws = RUNNER_RIG
    with pytest.raises(ValueError, match="slot 1"):
        FR.FrameRunner(ctx, 2, [(480, 640), (481, 640)], pixel_format=["rgb", "nv12"])
    with pytest.raises(ValueError, match="one per slot"):
        FR.FrameRunner(ctx, 3, [(480, 640), (240, 320)])
    with pytest.raises(ValueError, match="one per slot"):
        FR.FrameRunner(ctx, 2, (480, 640), pixel_format=["rgb", "nv12", "bgr"])
    runner = FR.FrameRunner(ctx, 4, hws, pixel_format=fmts)
    good = _blob_frames(fmts, hws, 0)
    with pytest.raises(ValueError, match="4 frames"):
        runner.submit(good[:3])
    with pytest.raises(ValueError, match="4 frames"):
        runner.submit(np.zeros((4, 480, 640, 3), np.uint8))
    bad = list(good)
    bad[2] = np.zeros((480, 640, 3), np.uint8)       # slot 2 is YUYV
    with pytest.raises(ValueError, match="slot 2"):
        runner.submit(bad)
    bad = list(good)
    bad[1] = good[1].astype(np.float32)
    with pytest.raises(TypeError, match="slot 1"):
        runner.submit(bad)
    bad = [torch.from_numpy(x).cuda() for x in good]
    bad[3] = torch.zeros((1280, 1080), dtype=torch.uint8, device="cuda").t()   # an I420 720x1280 frame's shape, not contiguous
    with pytest.raises(TypeError, match="slot 3"):
        runner.submit(bad)
    r = _host(runner.submit(good))                  # still serves after the refusals
    assert r["keypoints_frame"].shape == (4, 21, 2)
    del runner
    ctx.release_graphs()


def test_runner_on_poisoned_workspace_and_scratch(ctx):
    fmts, hws = RUNNER_RIG
    steps = [_blob_frames(fmts, hws, t, seed=41) for t in range(2)]

    def run():
        runner = FR.FrameRunner(ctx, 4, hws, pixel_format=fmts, draw=True, track=True, detect="slots")
        out = [_host(runner.submit(s)) for s in steps]
        del runner
        ctx.release_graphs()
        return out
    clean = run()
    for byte in (0x00, 0xFF):
        ctx.fill_scratch(byte)
        for t, (a, b) in enumerate(zip(run(), clean)):
            for k in b:
                if k == "frame_drawn":
                    for i in range(4):
                        _bits(a[k][i], b[k][i], "frame_drawn %d at step %d after a 0x%02X fill" % (i, t, byte))
                else:
                    _bits(a[k], b[k], "%s at step %d after a 0x%02X fill" % (k, t, byte))
    ctx.check_errors()


# ------------------------------------------------------------------------------------------------------------------ launch counting
# the rig entries and how this file counts their launches (tests/test_frames_rig_cpu.py checks that the tables cover _lib.RIG_SIGNATURES)
RIG_LAUNCH_CASES = {"h3d_frame_rig_plan": "plan", "h3d_resize_frames_rig": "resize"}
RIG_LAUNCH_EXCLUDED = {"h3d_frame_rig_query": "host only: builds the table without a context or a device"}

_CHILD = r"""
import json, sys
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile
sys.path.insert(0, sys.argv[2])
import frames_yuv_oracle as Y
from hand3d_b200 import runtime
ctx = runtime.default_context()
out = {}
for name, fmts, hws in json.loads(sys.argv[3]):
    frames = [torch.from_numpy(Y.random_frame(3, f, *hw)).cuda() for f, hw in zip(fmts, hws)]
    res = torch.empty((len(fmts), 240, 320, 3), dtype=torch.float32, device="cuda")
    ctx.frame_rig_plan(fmts, hws, 240, 320)
    torch.cuda.synchronize()
    calls = {"plan": lambda: ctx.frame_rig_plan(fmts, hws, 240, 320),
             "resize": lambda: ctx.resize_frames_rig(frames, 240, 320, True, out=res, pixel_formats=fmts)}
    for call, fn in calls.items():
        for _ in range(2):          # a session that recorded no CUDA event at all is repeated once
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                n0 = ctx.launch_count
                fn()
                torch.cuda.synchronize()
                n1 = ctx.launch_count
            cuda = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
            if cuda or n1 == n0:
                break
        out["%s-%s" % (name, call)] = {"launches": n1 - n0, "kernels": [n for n in cuda if "h3d::" in n]}
ctx.check_errors()
json.dump(out, open(sys.argv[1], "w"))
"""


def test_launch_count_equals_kernels_run(tmp_path):
    import json
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    rigs = [(k,) + RIGS[k] for k in ("3cams", "8cams")]
    path = str(tmp_path / "counts.json")
    r = subprocess.run([sys.executable, "-c", _CHILD, path, here, json.dumps(rigs)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=600, cwd=os.path.dirname(here))
    assert r.returncode == 0, r.stdout[-4000:]
    got = json.load(open(path))
    for name, fmts, _ in rigs:
        assert got[name + "-plan"]["launches"] == len(got[name + "-plan"]["kernels"]) == 0, got[name + "-plan"]
        res = got[name + "-resize"]
        assert res["launches"] == len(res["kernels"]) == len(set(fmts)), res
        assert all("resize_frames_rig_kernel" in k for k in res["kernels"]), res["kernels"]

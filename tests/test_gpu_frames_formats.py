"""Camera frames in other pixel formats on the device (h3d_resize_frames_fmt, h3d_convert_frames, hand3d_b200.frames with
pixel_format): every result equals, bit for bit, Pillow's BILINEAR resize of OpenCV's cvtColor conversion as tests/frames_yuv_oracle.py
restates them, and FrameRunner(pixel_format=f) equals FrameRunner() fed the converted RGB frames in every mode."""
import os

import numpy as np
import pytest
import torch

import frames_oracle as F
import frames_yuv_oracle as Y
from hand3d_b200 import _lib, runtime
from hand3d_b200 import frames as FR
from hand3d_b200 import weights as Wt

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_frames_yuv.npz")
NON_RGB = ("bgr",) + Y.YUV_FORMATS
# the frame sizes of test_gpu_frames.py made even, and its output sizes
FRAME_SIZES = [(480, 640), (720, 1280), (1080, 1920), (2160, 3840), (242, 322), (100, 78), (4, 6), (240, 320), (2, 2), (2, 700)]
OUT_SIZES = [(240, 320), (256, 256), (320, 320)]
# integer and non-integer factors both ways, and 1-pixel outputs
ODD_FACTORS = [((64, 96), (16, 24)), ((60, 90), (7, 11)), ((6, 14), (3, 5)), ((14, 18), (1, 1)), ((98, 90), (194, 178)), ((4096, 4), (1, 2)),
               ((4, 4096), (5, 3))]


@pytest.fixture(scope="module")
def ctx():
    c = runtime.Context()
    c.load_weights(Wt.synthetic_weights(0))
    yield c
    c.release_graphs()


def _batch(fmt, B, H, W, seed):
    return np.stack([Y.random_frame(seed + i, fmt, H, W) for i in range(B)])


def _ref(fmt, frames, h, w):
    return np.stack([Y.resize(fmt, f, h, w) for f in frames])


@pytest.mark.parametrize("fmt", NON_RGB)
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("frame_hw", FRAME_SIZES, ids=lambda s: "%dx%d" % s)
def test_resize_equals_restatement(ctx, fmt, B, frame_hw):
    fr = _batch(fmt, B, *frame_hw, seed=frame_hw[0] + 3 * frame_hw[1] + B)
    dev = torch.from_numpy(fr).cuda()
    rgb = [Y.to_rgb(fmt, f) for f in fr]
    for out_hw in OUT_SIZES:
        want = np.stack([F.imresize(x, *out_hw) for x in rgb])
        got = ctx.resize_frames(dev, *out_hw, normalize=False, pixel_format=fmt).cpu().numpy()
        np.testing.assert_array_equal(got, want, err_msg="to %dx%d" % out_hw)
        got = ctx.resize_frames(dev, *out_hw, normalize=True, pixel_format=fmt).cpu().numpy()
        np.testing.assert_array_equal(got.view(np.int32), F.normalize(want).view(np.int32), err_msg="normalised, to %dx%d" % out_hw)


@pytest.mark.parametrize("fmt", NON_RGB)
@pytest.mark.parametrize("frame_hw,out_hw", ODD_FACTORS, ids=lambda s: "%dx%d" % s)
def test_resize_odd_factors(ctx, fmt, frame_hw, out_hw):
    fr = _batch(fmt, 2, *frame_hw, seed=41)
    got = ctx.resize_frames(torch.from_numpy(fr).cuda(), *out_hw, normalize=False, pixel_format=fmt).cpu().numpy()
    np.testing.assert_array_equal(got, _ref(fmt, fr, *out_hw))


@pytest.mark.parametrize("fmt", NON_RGB)
@pytest.mark.parametrize("frame_hw", [(1080, 1920), (480, 640), (242, 322), (2, 700)], ids=lambda s: "%dx%d" % s)
def test_resize_batch32(ctx, fmt, frame_hw):
    fr = _batch(fmt, 32, *frame_hw, seed=11)
    got = FR.to_network_input(torch.from_numpy(fr).cuda(), pixel_format=fmt).cpu().numpy()
    np.testing.assert_array_equal(got.view(np.int32), F.normalize(_ref(fmt, fr, 240, 320)).view(np.int32))


@pytest.mark.parametrize("fmt", NON_RGB)
def test_identity_size_is_the_conversion(ctx, fmt):
    fr = _batch(fmt, 3, 240, 320, seed=51)
    dev = torch.from_numpy(fr).cuda()
    want = np.stack([Y.to_rgb(fmt, f) for f in fr])
    np.testing.assert_array_equal(ctx.resize_frames(dev, 240, 320, normalize=False, pixel_format=fmt).cpu().numpy(), want)
    np.testing.assert_array_equal(FR.to_rgb(dev, fmt).cpu().numpy(), want)
    np.testing.assert_array_equal(FR.to_rgb(dev[1], fmt).cpu().numpy(), want[1])           # one frame, unbatched
    np.testing.assert_array_equal(FR.to_network_input(dev[2], pixel_format=fmt).cpu().numpy().view(np.int32),
                                  F.normalize(want[2]).view(np.int32))


def test_rgb_entry_equals_resize_frames_and_bgr_equals_rgb(ctx):
    fr = torch.from_numpy(np.stack([F.frame(60 + i, 721, 1281) for i in range(3)])).cuda()
    for out_hw in OUT_SIZES:
        old = torch.empty((3,) + out_hw + (3,), dtype=torch.uint8, device="cuda")
        _lib.check(ctx.lib.h3d_resize_frames(ctx.h, fr.data_ptr(), 3, 721, 1281, out_hw[0], out_hw[1], 0, old.data_ptr(),
                                             torch.cuda.current_stream().cuda_stream), "h3d_resize_frames")
        new = ctx.resize_frames(fr, *out_hw, normalize=False, pixel_format="rgb")
        bgr = ctx.resize_frames(fr.flip(-1).contiguous(), *out_hw, normalize=False, pixel_format="bgr")
        torch.testing.assert_close(new, old, rtol=0, atol=0)
        torch.testing.assert_close(bgr, old, rtol=0, atol=0)
    np.testing.assert_array_equal(FR.to_rgb(fr, "rgb").cpu().numpy(), fr.cpu().numpy())


@pytest.mark.parametrize("fmt", NON_RGB)
@pytest.mark.parametrize("frame_hw", [(1080, 1920), (4096, 4096)], ids=lambda s: "%dx%d" % s)
def test_convert_equals_restatement(ctx, fmt, frame_hw):
    fr = _batch(fmt, 2, *frame_hw, seed=71)
    got = ctx.convert_frames(torch.from_numpy(fr).cuda(), fmt).cpu().numpy()
    np.testing.assert_array_equal(got, np.stack([Y.to_rgb(fmt, f) for f in fr]))


def test_device_equals_golden(ctx):
    z = np.load(GOLDEN)
    for i, (fmt, (H, W), seed) in enumerate(zip(z["formats"], z["sizes"], z["seeds"])):
        fmt = str(fmt)
        dev = torch.from_numpy(Y.random_frame(int(seed), fmt, int(H), int(W))).cuda()
        F.assert_equals_golden(FR.to_rgb(dev, fmt).cpu().numpy(), z, i)
        if H <= 512 and W <= 512:      # the identity resize is the conversion too
            F.assert_equals_golden(FR.imresize(FR.to_rgb(dev, fmt), (int(H), int(W))).cpu().numpy(), z, i)
            F.assert_equals_golden(ctx.resize_frames(dev[None], int(H), int(W), False, pixel_format=fmt)[0].cpu().numpy(), z, i)


@pytest.mark.parametrize("fmt", ["nv12", "yuyv"])
def test_past_2_gib(ctx, fmt):
    H = W = 4096
    B = 2 ** 31 // int(np.prod(Y.frame_shape(fmt, H, W))) + 2
    assert B * np.prod(Y.frame_shape(fmt, H, W)) > 2 ** 31
    g = torch.Generator(device="cuda").manual_seed(9)
    fr = torch.randint(0, 256, (B,) + Y.frame_shape(fmt, H, W), dtype=torch.uint8, device="cuda", generator=g)
    out = ctx.resize_frames(fr, 240, 320, normalize=False, pixel_format=fmt)
    for b in (0, B // 2, B - 1):
        host = fr[b].cpu().numpy()
        np.testing.assert_array_equal(out[b].cpu().numpy(), Y.resize(fmt, host, 240, 320), err_msg="image %d" % b)
        rgb = ctx.convert_frames(fr[b:b + 1], fmt)      # the full-size output of all B would be 4.4 GB; one image at its offset
        np.testing.assert_array_equal(rgb[0].cpu().numpy(), Y.to_rgb(fmt, host), err_msg="converted image %d" % b)
    del fr, out


def test_convert_past_2_gib_of_output(ctx):
    B, H, W = 44, 4096, 4096                    # the RGB output is 44 * 48 MiB > 2^31 bytes
    g = torch.Generator(device="cuda").manual_seed(10)
    fr = torch.randint(0, 256, (B,) + Y.frame_shape("i420", H, W), dtype=torch.uint8, device="cuda", generator=g)
    rgb = ctx.convert_frames(fr, "i420")
    for b in (0, B // 2, B - 1):
        np.testing.assert_array_equal(rgb[b].cpu().numpy(), Y.to_rgb("i420", fr[b].cpu().numpy()), err_msg="image %d" % b)
    del fr, rgb


# ---------------------------------------------------------------------------------------------------------------- FrameRunner
MODES = {"detect": {}, "track": {"track": True, "redetect_every": 3}, "slots": {"track": True, "detect": "slots", "redetect_every": 2}}


def _keys(res):
    return [k for k in res if k != "detected"]


@pytest.mark.parametrize("fmt", NON_RGB)
@pytest.mark.parametrize("mode", list(MODES))
def test_frame_runner_equals_rgb_runner(ctx, fmt, mode):
    B, frame_hw = 2, (480, 640)
    steps = [_batch(fmt, B, *frame_hw, seed=300 + 5 * t) for t in range(4)]
    rgb_steps = [np.stack([Y.to_rgb(fmt, f) for f in s]) for s in steps]
    got, want = [], []
    for pf, seq, out in ((fmt, steps, got), ("rgb", rgb_steps, want)):
        runner = FR.FrameRunner(ctx, B, frame_hw, draw=True, pixel_format=pf, **MODES[mode])
        assert runner.frame_hw == frame_hw
        for t, s in enumerate(seq):             # host and CUDA input alternately
            r = runner.submit(s if t % 2 == 0 else torch.from_numpy(s).cuda())
            out.append({k: (r[k].cpu().numpy() if isinstance(r[k], torch.Tensor) else r[k]) for k in _keys(r)} | {"detected": r.get("detected")})
        del runner
        ctx.release_graphs()
    for t, (g, w) in enumerate(zip(got, want)):
        assert sorted(g) == sorted(w)
        assert g["frame_drawn"].shape == (B,) + frame_hw + (3,)
        for k in w:
            np.testing.assert_array_equal(g[k], w[k], err_msg="%s at step %d" % (k, t))


def test_frame_runner_stream_and_device_step_never_syncs(ctx):
    B, frame_hw, fmt = 2, (480, 640), "nv12"
    runner = FR.FrameRunner(ctx, B, frame_hw, draw=True, pixel_format=fmt)
    frs = [_batch(fmt, B, *frame_hw, seed=400 + i) for i in range(3)]
    dev = [torch.from_numpy(f).cuda() for f in frs]
    torch.cuda.synchronize()
    outs = []
    torch.cuda.set_sync_debug_mode("error")
    try:
        for d in dev:                                   # refills the captured buffers and replays
            r = runner.submit(d)
            outs.append({k: v.clone() for k, v in r.items()})
    finally:
        torch.cuda.set_sync_debug_mode(0)
    streamed = list(runner.stream(iter(frs)))
    del runner
    ctx.release_graphs()
    ref = FR.FrameRunner(ctx, B, frame_hw, draw=True)
    for i, f in enumerate(frs):
        w = ref.submit(np.stack([Y.to_rgb(fmt, x) for x in f]))
        for k in w:
            np.testing.assert_array_equal(outs[i][k].cpu().numpy(), w[k].cpu().numpy(), err_msg="%s at step %d" % (k, i))
            np.testing.assert_array_equal(streamed[i][k], w[k].cpu().numpy(), err_msg="streamed %s at step %d" % (k, i))
    del ref
    ctx.release_graphs()


def test_poisoned_workspace_and_scratch(ctx):
    fr = {f: torch.from_numpy(_batch(f, 3, 482, 642, seed=90)).cuda() for f in NON_RGB}
    ctx.ensure_workspace(3, 240, 320)

    def run():
        return [ctx.resize_frames(fr[f], 240, 320, normalize=n, pixel_format=f).cpu() for f in NON_RGB for n in (False, True)] + \
               [ctx.convert_frames(fr[f], f).cpu() for f in NON_RGB]
    clean = run()
    for byte in (0x00, 0xFF, 0x7F):
        ctx.fill_scratch(byte)
        for a, b in zip(run(), clean):
            assert torch.equal(a, b), "a result changed after a 0x%02X fill" % byte
    ctx.check_errors()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def test_refusals_before_any_launch(ctx):
    src = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    out = torch.full((1 << 20,), 0xA5, dtype=torch.uint8, device="cuda")
    bad = [  # (format, B, H, W, out_h, out_w)
        (_lib.PIXEL_FORMATS["nv12"], 1, 5, 8, 4, 4), (_lib.PIXEL_FORMATS["nv12"], 1, 8, 5, 4, 4), (_lib.PIXEL_FORMATS["i420"], 1, 7, 8, 4, 4),
        (_lib.PIXEL_FORMATS["i420"], 1, 8, 9, 4, 4), (_lib.PIXEL_FORMATS["yuyv"], 1, 8, 7, 4, 4), (_lib.PIXEL_FORMATS["yuyv"], 1, 8, 1, 4, 4),
        (5, 1, 8, 8, 4, 4), (-1, 1, 8, 8, 4, 4), (_lib.PIXEL_FORMATS["nv12"], 1, 4098, 8, 4, 4), (_lib.PIXEL_FORMATS["yuyv"], 1, 8, 4098, 4, 4),
        (_lib.PIXEL_FORMATS["bgr"], 1, 8, 8, 513, 4), (_lib.PIXEL_FORMATS["nv12"], 1, 8, 8, 4, 0), (_lib.PIXEL_FORMATS["nv12"], 0, 8, 8, 4, 4),
        (_lib.PIXEL_FORMATS["nv12"], 1, 0, 8, 4, 4),
    ]
    launches = ctx.launch_count
    for fmt, B, H, W, h, w in bad:
        rc = ctx.lib.h3d_resize_frames_fmt(ctx.h, src.data_ptr(), fmt, B, H, W, h, w, 0, out.data_ptr(), _stream())
        assert rc == _lib.EINVAL, (fmt, B, H, W, h, w)
        if h > 0 and w > 0 and h <= 512 and w <= 512:   # the conversion has no output size
            rc = ctx.lib.h3d_convert_frames(ctx.h, src.data_ptr(), fmt, B, H, W, out.data_ptr(), _stream())
            assert rc == _lib.EINVAL, ("convert", fmt, B, H, W)
    assert ctx.lib.h3d_resize_frames_fmt(ctx.h, src.data_ptr(), 2, 1, 8, 8, 4, 4, 2, out.data_ptr(), _stream()) == _lib.EINVAL  # normalize
    assert ctx.lib.h3d_convert_frames(ctx.h, None, 2, 1, 8, 8, out.data_ptr(), _stream()) == _lib.EINVAL
    torch.cuda.synchronize()
    assert ctx.launch_count == launches
    assert bool((out == 0xA5).all()), "a refused call wrote its output"
    good = torch.zeros((1, 12, 8), dtype=torch.uint8, device="cuda")       # an 8x8 NV12 frame
    for t, fmt, exc in [(good.float(), "nv12", TypeError), (good.cpu(), "nv12", RuntimeError), (good, "rgba", ValueError),
                        (torch.zeros((1, 13, 8), dtype=torch.uint8, device="cuda"), "nv12", ValueError),
                        (torch.zeros((1, 8, 8, 3), dtype=torch.uint8, device="cuda"), "yuyv", ValueError),
                        (torch.zeros((1, 8, 8, 2), dtype=torch.uint8, device="cuda"), "bgr", ValueError),
                        (torch.zeros((1, 24, 16), dtype=torch.uint8, device="cuda")[:, :, ::2], "i420", ValueError),
                        (torch.zeros((1, 12, 7), dtype=torch.uint8, device="cuda"), "nv12", RuntimeError)]:
        with pytest.raises(exc):
            ctx.resize_frames(t, 4, 4, False, pixel_format=fmt)
        with pytest.raises(exc):
            ctx.convert_frames(t, fmt)
    with pytest.raises(ValueError):
        FR.FrameRunner(ctx, 1, (7, 8), pixel_format="nv12")
    runner = FR.FrameRunner(ctx, 1, (8, 8), pixel_format="nv12")
    with pytest.raises(ValueError):
        runner.submit(np.zeros((1, 8, 8, 3), np.uint8))
    del runner
    ctx.release_graphs()

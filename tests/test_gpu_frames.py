"""Camera frames on the device (hand3d_b200.frames, h3d_resize_frames): the resize equals the numpy restatement of Pillow's BILINEAR and
the Pillow golden bit for bit, the fused normalisation equals run.py's float64 path, and FrameRunner equals the pipeline run on
host-prepared input, eagerly and through its overlapped stream."""
import os

import numpy as np
import pytest
import torch

import frames_oracle as F
from hand3d_b200 import frames as FR
from hand3d_b200 import runtime
from hand3d_b200 import weights as Wt

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_frames_pil.npz")
FRAME_SIZES = [(480, 640), (720, 1280), (1080, 1920), (2160, 3840), (241, 321), (100, 77), (3, 5), (240, 320), (1, 1), (2, 700)]
OUT_SIZES = [(240, 320), (256, 256), (320, 320)]


@pytest.fixture(scope="module")
def ctx():
    c = runtime.Context()
    c.load_weights(Wt.synthetic_weights(0))
    yield c
    c.release_graphs()


def _batch(B, H, W, seed):
    return np.stack([F.frame(seed + i, H, W) for i in range(B)])


def _ref(frames, h, w):
    return np.stack([F.imresize(f, h, w) for f in frames])


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("frame_hw", FRAME_SIZES, ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("out_hw", OUT_SIZES, ids=lambda s: "to%dx%d" % s)
def test_resize_equals_restatement(ctx, B, frame_hw, out_hw):
    fr = _batch(B, *frame_hw, seed=frame_hw[0] + 3 * frame_hw[1] + B)
    got = ctx.resize_frames(torch.from_numpy(fr).cuda(), *out_hw, normalize=False).cpu().numpy()
    np.testing.assert_array_equal(got, _ref(fr, *out_hw))


@pytest.mark.parametrize("frame_hw", [(1080, 1920), (480, 640), (241, 321), (2, 700)], ids=lambda s: "%dx%d" % s)
def test_resize_batch32(ctx, frame_hw):
    fr = _batch(32, *frame_hw, seed=11)
    got = ctx.resize_frames(torch.from_numpy(fr).cuda(), 240, 320, normalize=False).cpu().numpy()
    np.testing.assert_array_equal(got, _ref(fr, 240, 320))


def test_resize_equals_pillow_golden(ctx):
    z = np.load(GOLDEN)
    for i, (H, W, h, w) in enumerate(z["cases"]):
        fr = F.frame(7000 + i, int(H), int(W))
        got = FR.imresize(torch.from_numpy(fr).cuda(), (int(h), int(w))).cpu().numpy()
        F.assert_equals_golden(got, z, i)


def test_resize_past_2_gib(ctx):
    B, H, W = 43, 4096, 4096                 # 43 * 4096 * 4096 * 3 bytes > 2^31
    assert B * H * W * 3 > 2 ** 31
    g = torch.Generator(device="cuda").manual_seed(5)
    fr = torch.randint(0, 256, (B, H, W, 3), dtype=torch.uint8, device="cuda", generator=g)
    out = ctx.resize_frames(fr, 240, 320, normalize=False)
    for b in (0, 21, B - 1):
        np.testing.assert_array_equal(out[b].cpu().numpy(), F.imresize(fr[b].cpu().numpy(), 240, 320), err_msg="image %d" % b)
    del fr


@pytest.mark.parametrize("frame_hw", [(1080, 1920), (480, 640), (3, 5), (240, 320)], ids=lambda s: "%dx%d" % s)
def test_to_network_input_bit_exact(ctx, frame_hw):
    fr = _batch(3, *frame_hw, seed=21)
    got = FR.to_network_input(torch.from_numpy(fr).cuda()).cpu().numpy()
    want = F.normalize(_ref(fr, 240, 320))
    np.testing.assert_array_equal(got.view(np.int32), want.view(np.int32))
    allcodes = np.broadcast_to(np.arange(256, dtype=np.uint8)[None, :, None], (240, 256, 3)).copy()   # an identity resize of every code
    got = FR.to_network_input(torch.from_numpy(allcodes).cuda(), size=(240, 256)).cpu().numpy()
    np.testing.assert_array_equal(got.view(np.int32), F.normalize(allcodes).view(np.int32))


def test_imresize_numpy_and_ranks(ctx):
    fr = F.frame(3, 241, 321)
    out = FR.imresize(fr, (240, 320))
    assert isinstance(out, np.ndarray) and out.dtype == np.uint8
    np.testing.assert_array_equal(out, F.imresize(fr, 240, 320))
    np.testing.assert_array_equal(FR.imresize(fr, 50), F.imresize(fr, 120, 160))        # scipy: an int is a percentage
    np.testing.assert_array_equal(FR.imresize(fr, 0.5), F.imresize(fr, 120, 160))       # a float a fraction
    t = FR.imresize(torch.from_numpy(fr).cuda(), (240, 320))
    assert t.is_cuda and tuple(t.shape) == (240, 320, 3)


def test_frame_coords_device(ctx):
    c = np.array([[[0.0, 0.0], [239.0, 319.0], [119.5, 159.5], [10.0, 20.0]]])
    got = FR.frame_coords(torch.from_numpy(c).cuda(), (1080, 1920))
    assert got.dtype == torch.float64 and got.is_cuda
    np.testing.assert_array_equal(got.cpu().numpy(), [[[1.75, 2.5], [1077.25, 1916.5], [539.5, 959.5], [46.75, 122.5]]])
    np.testing.assert_array_equal(FR.frame_coords(c, (480, 640)), F.frame_coords(c, (480, 640)))


def _eager(ctx, fr, hs, frame_hw):
    """The pipeline on the host-prepared input (restated resize + run.py's normalisation on the host)."""
    img = torch.from_numpy(np.ascontiguousarray(F.normalize(_ref(fr, 240, 320)))).cuda()
    r = ctx.pipeline(img, torch.from_numpy(np.asarray(hs, np.float32)).cuda(), True, outputs="keypoints")
    r = {k: r[k].cpu().numpy() for k in ("keypoints_uv", "keypoint_coord3d", "center", "scale_crop")}
    kp = (r["keypoints_uv"].astype(np.float64) - 128) / r["scale_crop"].astype(np.float64).reshape(-1, 1, 1) \
        + r["center"].astype(np.float64).reshape(-1, 1, 2)        # trafo_coords(..., 256)
    r["keypoints_frame"] = F.frame_coords(kp, frame_hw)
    return r


def _assert_same(got, want, what=""):
    for k, v in want.items():
        g = got[k].cpu().numpy() if isinstance(got[k], torch.Tensor) else got[k]
        np.testing.assert_array_equal(g, v, err_msg="%s %s" % (what, k))


@pytest.mark.parametrize("frame_hw", [(1080, 1920), (480, 640)], ids=lambda s: "%dx%d" % s)
def test_frame_runner_equals_pipeline(ctx, frame_hw):
    B = 2
    runner = FR.FrameRunner(ctx, B, frame_hw)
    fr = _batch(B, *frame_hw, seed=31)
    hs = [[1.0, 0.0]] * B
    want = _eager(ctx, fr, hs, frame_hw)
    _assert_same(runner.submit(fr), want, "host")
    _assert_same(runner.submit(torch.from_numpy(fr).cuda()), want, "device")
    del runner
    ctx.release_graphs()


def test_frame_runner_stream_equals_eager(ctx):
    B, frame_hw = 2, (480, 640)
    runner = FR.FrameRunner(ctx, B, frame_hw)
    batches = [(_batch(B, *frame_hw, seed=100 + 7 * i), np.array([[1.0, 0.0], [0.0, 1.0]] if i % 2 else [[0.0, 1.0]] * B, np.float32))
               for i in range(7)]
    got = list(runner.stream(iter(batches)))
    assert len(got) == len(batches)
    for i, ((fr, hs), g) in enumerate(zip(batches, got)):
        _assert_same(g, _eager(ctx, fr, hs, frame_hw), "batch %d" % i)
    del runner
    ctx.release_graphs()


def test_frame_runner_device_step_never_syncs(ctx):
    B, frame_hw = 2, (480, 640)
    runner = FR.FrameRunner(ctx, B, frame_hw)
    frs = [_batch(B, *frame_hw, seed=200 + i) for i in range(3)]
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
    for i, f in enumerate(frs):
        _assert_same(outs[i], _eager(ctx, f, [[1.0, 0.0]] * B, frame_hw), "step %d" % i)
    del runner
    ctx.release_graphs()


def test_refusals(ctx):
    good = torch.zeros((1, 8, 8, 3), dtype=torch.uint8, device="cuda")
    with pytest.raises(TypeError):
        ctx.resize_frames(good.float(), 4, 4, False)
    for c in (1, 4):
        with pytest.raises(ValueError):
            ctx.resize_frames(torch.zeros((1, 8, 8, c), dtype=torch.uint8, device="cuda"), 4, 4, False)
    with pytest.raises(ValueError):
        ctx.resize_frames(torch.zeros((1, 8, 16, 3), dtype=torch.uint8, device="cuda")[:, :, ::2], 4, 4, False)
    with pytest.raises(RuntimeError):
        ctx.resize_frames(good.cpu(), 4, 4, False)
    for shape, out in [((1, 0, 8, 3), (4, 4)), ((1, 8, 0, 3), (4, 4)), ((0, 8, 8, 3), (4, 4)), ((1, 4097, 1, 3), (4, 4)),
                       ((1, 1, 4097, 3), (4, 4))]:
        with pytest.raises(RuntimeError):
            ctx.resize_frames(torch.zeros(shape, dtype=torch.uint8, device="cuda"), *out, False)
    for out in [(0, 4), (4, 0), (513, 4), (4, 513)]:
        with pytest.raises(RuntimeError):
            ctx.resize_frames(good, *out, False)
    with pytest.raises(ValueError):
        FR.imresize(np.zeros((8, 8, 3), np.uint8), (4, 4), interp="nearest")
    with pytest.raises(ValueError):
        FR.imresize(np.zeros((8, 8, 3), np.uint8), (4, 4), mode="L")
    with pytest.raises(TypeError):
        FR.imresize(np.zeros((8, 8, 3), np.float32), (4, 4))
    with pytest.raises(ValueError):
        FR.imresize(np.zeros((8, 8), np.uint8), (4, 4))
    with pytest.raises(RuntimeError):
        FR.to_network_input(good.cpu())
    with pytest.raises(TypeError):
        FR.FrameRunner(ctx, 1, (8, 8)).submit(np.zeros((1, 8, 8, 3), np.float32))
    ctx.release_graphs()

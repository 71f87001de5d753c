"""Per-slot re-detection (h3d_track_step_slots, Context.track_step_slots, FrameRunner(track=True, detect="slots")): a slots step
equals, slot by slot and bit for bit, a detect step for the slots it selects and a track step for the others; the limits n = 0 and
n = B; the launches it adds; poisoned workspaces; graph replay; FrameRunner's per-slot policy on a synthetic sequence (against the
restatement of tests/track_slots_oracle.py); and the argument checks."""
import gc

import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import track_oracle as T
import track_slots_oracle as S
from hand3d_b200 import _lib, runtime
from hand3d_b200 import weights as Wt
from hand3d_b200.frames import FrameRunner

pytestmark = pytest.mark.gpu
W_SEG = Wt.synthetic_weights(0, seg_shift=0.15)   # blob images give varied masks with these
F = np.float32
OUT_KEYS = ("image_crop", "scale_crop", "center", "keypoints_scoremap", "keypoint_coord3d", "keypoints_uv")
STATE_KEYS = ("center", "scale", "score", "lost")


def _context():
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


@pytest.fixture(scope="module")
def ctx():
    yield from _context()


@pytest.fixture(scope="module")
def wide():
    """Contexts for the batches of 32 and more, one frame size at a time.  A workspace grows to the largest batch and the largest frame
    it has seen, so each frame size gets a context of its own, and the previous one is destroyed before the next is made."""
    held = {}

    def get(hw):
        if hw not in held:
            for gen, _ in held.values():
                gen.close()
            held.clear()
            gen = _context()
            held[hw] = (gen, next(gen))
        return held[hw][1]

    yield get
    for gen, _ in held.values():
        gen.close()


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _host(r):
    return {k: v.cpu().numpy() for k, v in r.items() if isinstance(v, torch.Tensor)}


def _state_host(st):
    return {"center": st.center.cpu().numpy(), "scale": st.scale.cpu().numpy(), "score": st.score.cpu().numpy(),
            "lost": st.lost.cpu().numpy()}


def _copy_state(st):
    c = runtime.TrackState(st.B, st.buffer.device)
    c.buffer.copy_(st.buffer)
    return c


def _bits_equal(got, want, what):
    """Bit-equal, except that any NaN equals any NaN."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    if got.dtype.kind == "f":
        gn, wn = np.isnan(got), np.isnan(want)
        np.testing.assert_array_equal(gn, wn, err_msg="%s: NaN positions" % what)
        got, want = np.where(gn, 0, got).astype(got.dtype), np.where(wn, 0, want).astype(want.dtype)
        got, want = got.view(np.int32), want.view(np.int32)
    np.testing.assert_array_equal(got, want, err_msg=what)


def _case(ctx, precision, B, H, W, seed):
    """Images, hand sides and a state whose crops are near the detected ones (as the previous frame's key-points would give)."""
    ctx.set_precision(precision)
    img = _dev(Wt.synthetic_blob_images(B, H, W, seed=seed))
    hs = _dev(Wt.synthetic_hand_side(B, seed=seed + 1))
    st = runtime.TrackState(B)
    det = _host(ctx.track_step(img, hs, st, True, outputs="keypoints"))
    rng = np.random.default_rng(seed)
    st.center.copy_(_dev(det["center"] + rng.uniform(-6, 6, (B, 2)).astype(F)))
    st.scale.copy_(_dev(det["scale_crop"].reshape(B) * rng.uniform(0.9, 1.1, B).astype(F)))
    return img, hs, st


def _pattern(B, seed, n_sel=None):
    """(lost, force) int32 [B]: a random selection, both flags set on some slots, or exactly n_sel slots lost."""
    rng = np.random.default_rng(seed)
    if n_sel is not None:
        lost = np.zeros(B, np.int32)
        lost[rng.permutation(B)[:n_sel]] = 1
        return lost, np.zeros(B, np.int32)
    return (rng.random(B) < 0.3).astype(np.int32), (rng.random(B) < 0.2).astype(np.int32)


def _slots_vs_full(ctx, img, hs, st, lost, force, min_score=None):
    """Runs the slots step, a detect step and a track step from copies of the same state; returns the three (outputs, state after)."""
    st.lost.copy_(_dev(lost))
    sa, sd, stk = _copy_state(st), _copy_state(st), _copy_state(st)
    got = _host(ctx.track_step_slots(img, hs, sa, force=None if force is None else _dev(force), min_score=min_score))
    det = _host(ctx.track_step(img, hs, sd, True, min_score=min_score))
    trk = _host(ctx.track_step(img, hs, stk, False, min_score=min_score))
    return (got, _state_host(sa)), (det, _state_host(sd)), (trk, _state_host(stk))


def _check_composed(got, det, trk, sel):
    (g, gs), (d, ds), (t, ts) = got, det, trk
    np.testing.assert_array_equal(g["track_detected"], sel.astype(bool))
    for b in range(len(sel)):
        ref, ref_s = (d, ds) if sel[b] else (t, ts)
        for k in OUT_KEYS:
            _bits_equal(g[k][b], ref[k][b], "%s of slot %d (selected %d)" % (k, b, sel[b]))
        for k in STATE_KEYS:
            _bits_equal(gs[k][b], ref_s[k][b], "state %s of slot %d (selected %d)" % (k, b, sel[b]))


# B = 160 at 600x800 is left out: its workspace (about 80 GB) does not fit beside the rest on an 80 GB card
COMPOSE = ([(B, 240, 320) for B in (1, 3, 32, 160)] + [(B, 320, 320) for B in (1, 3, 32, 160)] +
           [(B, 600, 800) for B in (1, 3, 32)])


@pytest.mark.parametrize("precision", ["bf16x3", "fp16"])
@pytest.mark.parametrize("B,H,W", COMPOSE)
def test_slots_step_composes_detect_and_track(ctx, wide, precision, B, H, W):
    ctx = wide((H, W)) if B >= 32 else ctx
    img, hs, st = _case(ctx, precision, B, H, W, seed=B + H + W)
    lost, force = _pattern(B, seed=B * 3 + H)
    sel = S.select(lost, force)[2]
    got, det, trk = _slots_vs_full(ctx, img, hs, st, lost, force)
    _check_composed(got, det, trk, sel)


@pytest.mark.parametrize("precision", ["fp16x3", "bf16", "fp32_ffma", "fp16_f8c"])
def test_slots_step_composes_in_every_mode(ctx, precision):
    B, H, W = 5, 240, 320
    img, hs, st = _case(ctx, precision, B, H, W, seed=41)
    lost, force = np.array([0, 1, 0, 0, 1], np.int32), np.array([0, 0, 1, 0, 1], np.int32)
    got, det, trk = _slots_vs_full(ctx, img, hs, st, lost, force)
    _check_composed(got, det, trk, S.select(lost, force)[2])


@pytest.mark.parametrize("switch", ["no_pool_fusion", "no_seg_fusion"])
def test_slots_step_composes_with_unfused_kernels(ctx, switch):
    """no_pool_fusion: the counted stand-alone max-pool of the split planes; no_seg_fusion: the counted stand-alone x8 up-sampling
    followed by the unfused post-processing, in the detect step and in the slots step alike."""
    ctx.set_tuning(switch, 1)
    try:
        B, H, W = 5, 240, 320
        img, hs, st = _case(ctx, "bf16x3", B, H, W, seed=43)
        lost, force = np.array([1, 0, 0, 1, 0], np.int32), np.array([0, 0, 1, 0, 0], np.int32)
        got, det, trk = _slots_vs_full(ctx, img, hs, st, lost, force)
        _check_composed(got, det, trk, S.select(lost, force)[2])
    finally:
        ctx.set_tuning(switch, 0)


def _a(x, n):
    return -(-x // n) * n


def _seg_regions(B, H, W, precision):
    """{name: (byte offset, bytes per compact image)} of what HandSegNet and the mask post-processing write in a workspace laid out for
    (B, H, W): api.cu's layout() (1024-byte aligned arena) and build_handsegnet()'s two ping-pong slots (one or two planes each)."""
    off, o = 0, {}

    def alloc(name, nbytes):
        nonlocal off
        off = _a(off, 1024)
        o[name] = off
        off += nbytes

    Ww = (W + 31) // 32
    Hc, Wc = max(H, 256), max(W, 256)
    for name, nbytes in [("hand_scoremap", B * H * W * 8), ("image_crop", B * 256 * 256 * 12), ("kp_scoremap", B * 256 * 256 * 84),
                         ("center", B * 8), ("scale", B * 4), ("crop_size", B * 4), ("coord3d", B * 63 * 4), ("kp_uv", B * 42 * 4),
                         ("seg_scratch", _a(B * 8, 256) + _a(B * H * Ww * 4, 256)), ("argmax", _a(B * 21 * 8, 256)),
                         ("seg_low", B * (H // 8) * (W // 8) * 8)] + [("s%d" % i, B * (Hc // 8) * (Wc // 8) * 84) for i in range(3)]:
        alloc(name, nbytes)
    seg_off = _a(off, 1024)
    se = B * H * W * 64                                   # elements of one slot
    regions = {"hand_scoremap": (o["hand_scoremap"], H * W * 8), "crop_size": (o["crop_size"], 4),
               "mask_bits": (o["seg_scratch"] + _a(B * 8, 256), H * Ww * 4), "seg_low": (o["seg_low"], (H // 8) * (W // 8) * 8)}
    for k in range(2):
        slot = seg_off + k * _a(se * 4, 1024)
        if precision == "fp32_ffma":
            regions["slot%d" % k] = (slot, H * W * 64 * 4)
        else:                                             # 3-pass split planes: hi, then lo at the next 1024 bytes
            regions["slot%d_hi" % k] = (slot, H * W * 64 * 2)
            regions["slot%d_lo" % k] = (slot + _a(se * 2, 1024), H * W * 64 * 2)
    return regions


@pytest.mark.parametrize("precision,H,W", [("bf16x3", 240, 320), ("fp32_ffma", 240, 320), ("bf16x3", 600, 800)])
def test_counted_pass_leaves_the_other_compact_images_untouched(precision, H, W):
    """After a sentinel fill of the workspace, a slots step with n selected slots writes HandSegNet's activations, its low-resolution
    head, the hand score map, the mask bits and the crop sizes of compact images < n only.  n = 0 leaves every one of those regions
    untouched, so a kernel of the counted plan that ignored the count would show; n = 1 (slot 1) writes compact image 0 and not 1, 2;
    n = B writes every image (which also checks the offsets).  A context of its own keeps the layout at exactly (3, H, W)."""
    B, SENT = 3, 0x7B
    gen = _context()
    c = next(gen)
    try:
        img, hs, st = _case(c, precision, B, H, W, seed=29)
        assert c._ws_key == (B, H, W)
        base = _a(c._ws.data_ptr(), 1024) - c._ws.data_ptr()
        regions = _seg_regions(B, H, W, precision)

        def run(force):
            s = _copy_state(st)
            s.lost.zero_()
            c.fill_scratch(SENT)
            c.track_step_slots(img, hs, s, force=_dev(np.array(force, np.int32)))
            torch.cuda.synchronize()
            return {k: c._ws[base + o: base + o + B * n].cpu().numpy().reshape(B, n) for k, (o, n) in regions.items()}

        for force, n_sel in (([0, 0, 0], 0), ([0, 1, 0], 1), ([1, 1, 1], 3)):
            got = run(force)
            for k, v in got.items():
                untouched = (v == SENT).all(axis=1)
                want = np.array([i >= n_sel for i in range(B)])
                if k.startswith("slot") and n_sel == B:
                    # a slot's chunk of H * W * 64 elements per image is what its largest layer (conv1_1 / conv1_2) may write; with
                    # the max-pool fused into conv1_2 the second slot only ever holds [B, H/2, W/2, 64] and smaller, so it never reaches
                    # the chunks of images 1 and 2: with every slot selected, only image 0's chunk must have been written
                    untouched, want = untouched[:1], want[:1]
                np.testing.assert_array_equal(untouched, want, err_msg="%s: compact images left at the sentinel with n = %d" % (k, n_sel))
    finally:
        gen.close()


@pytest.mark.parametrize("precision", ["bf16x3", "fp16"])
def test_limits_none_and_all(ctx, precision):
    B, H, W = 4, 240, 320
    img, hs, st = _case(ctx, precision, B, H, W, seed=7)
    zero = np.zeros(B, np.int32)
    got, det, trk = _slots_vs_full(ctx, img, hs, st, zero, None)          # n = 0: a track step
    for k in OUT_KEYS:
        _bits_equal(got[0][k], trk[0][k], k)
    for k in STATE_KEYS:
        _bits_equal(got[1][k], trk[1][k], "state " + k)
    assert not got[0]["track_detected"].any()
    got, det, trk = _slots_vs_full(ctx, img, hs, st, zero, np.ones(B, np.int32))   # n = B: a detect step
    for k in OUT_KEYS:
        _bits_equal(got[0][k], det[0][k], k)
    for k in STATE_KEYS:
        _bits_equal(got[1][k], det[1][k], "state " + k)
    assert got[0]["track_detected"].all()


def test_launches_add_select_counted_plan_and_merge(ctx):
    ctx.set_precision("bf16x3")
    B, H, W = 3, 240, 320
    img, hs, st = _case(ctx, "bf16x3", B, H, W, seed=9)
    ctx.track_step_slots(img, hs, st)                        # warm-up: the counted plan is built

    def launches(fn):
        torch.cuda.synchronize()
        n0 = ctx.launch_count
        fn()
        torch.cuda.synchronize()
        return ctx.launch_count - n0

    det = launches(lambda: ctx.track_step(img, hs, st, True, outputs="keypoints"))
    trk = launches(lambda: ctx.track_step(img, hs, st, False, outputs="keypoints"))
    for n_sel in (0, 1, B):
        st.lost.copy_(_dev(_pattern(B, 1, n_sel)[0]))
        slots = launches(lambda: ctx.track_step_slots(img, hs, st, outputs="keypoints"))
        print("launches: detect %d, track %d, slots (n = %d) %d" % (det, trk, n_sel, slots))
        assert slots - trk == 1 + (det - trk) + 1             # select, HandSegNet + mask post-processing (counted), merge


@pytest.mark.parametrize("H,W", [(240, 320), (600, 800)])
def test_poisoned_workspace_gives_the_same_bits(ctx, H, W):
    B = 3
    img, hs, st = _case(ctx, "bf16x3", B, H, W, seed=13)
    lost, force = np.array([1, 0, 0], np.int32), np.array([0, 0, 1], np.int32)
    st.lost.copy_(_dev(lost))
    runs = []
    for byte in (0x00, 0xFF, 0x7B):
        s = _copy_state(st)
        ctx.fill_scratch(byte)
        r = _host(ctx.track_step_slots(img, hs, s, force=_dev(force)))
        runs.append((r, _state_host(s)))
    for (r, s) in runs[1:]:
        for k in runs[0][0]:
            _bits_equal(r[k], runs[0][0][k], k)
        for k in STATE_KEYS:
            _bits_equal(s[k], runs[0][1][k], "state " + k)


def test_graph_replay_equals_eager(ctx):
    ctx.set_precision("bf16x3")
    B, H, W = 4, 240, 320
    img, hs, st = _case(ctx, "bf16x3", B, H, W, seed=17)
    force = _dev(np.array([0, 1, 0, 0], np.int32))
    st.lost.copy_(_dev(np.array([1, 0, 0, 0], np.int32)))
    st0 = _copy_state(st)
    eager = []
    se = _copy_state(st0)
    for _ in range(3):
        eager.append((_host(ctx.track_step_slots(img, hs, se, force=force)), _state_host(se)))
    sg = _copy_state(st0)
    ctx.track_step_slots(img, hs, _copy_state(st0), force=force)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        res = ctx.track_step_slots(img, hs, sg, force=force)
    ctx._graphs_captured = getattr(ctx, "_graphs_captured", 0) + 1
    try:
        sg.buffer.copy_(st0.buffer)
        for t in range(3):
            g.replay()
            r, s = _host(res), _state_host(sg)
            for k in eager[t][0]:
                _bits_equal(r[k], eager[t][0][k], "%s at replay %d" % (k, t))
            for k in STATE_KEYS:
                _bits_equal(s[k], eager[t][1][k], "state %s at replay %d" % (k, t))
    finally:
        del g
        ctx.release_graphs()


def _uint8(img):
    return np.clip(np.round((img + 0.5) * 255.0), 0, 255).astype(np.uint8)


def _sequence(n, noise_at, H=240, W=320):
    """Three streams of a blob image shifted (2, 3) px per frame; stream 0 gets a faint-noise frame at noise_at."""
    base = _uint8(Wt.synthetic_blob_images(3, H, W, seed=21))
    rng = np.random.default_rng(22)
    frames = []
    for t in range(n):
        f = np.stack([np.roll(base[b], (2 * t, 3 * t), axis=(0, 1)) for b in range(3)])
        if t == noise_at:
            f[0] = rng.integers(126, 131, (H, W, 3), dtype=np.uint8)
        frames.append(f)
    return frames


def _check_slots_policy(res, every, min_score, margin):
    """The restatement's per-slot choice and crops, from the device's own key-points and scores, step by step."""
    B = len(res[0]["center"])
    state = T.new_state(B)
    for t, r in enumerate(res):
        force = S.redetect_force(B, every, t) if every is not None else None
        _, _, want = S.select(state["lost"], force)
        np.testing.assert_array_equal(r["track_detected"], want.astype(bool), err_msg="selection at step %d" % t)
        for b in range(B):
            if not want[b]:
                _bits_equal(r["center"][b], state["center"][b], "center of slot %d at step %d" % (b, t))
                _bits_equal(r["scale_crop"][b, 0], state["scale"][b], "scale of slot %d at step %d" % (b, t))
        for b in range(B):
            c, s, fb = T.next_crop(r["keypoints_uv"][b], r["center"][b], r["scale_crop"][b, 0], margin)
            lost = fb or (min_score is not None and not (r["track_score"][b] >= F(min_score)))
            assert bool(r["track_lost"][b]) == lost, (t, b)
            state["lost"][b] = int(lost)
            if not lost:
                state["center"][b], state["scale"][b] = c, s


def test_frame_runner_slots_redetects_only_the_lost_slot_one_step_later(ctx):
    ctx.set_precision("bf16x3")
    n, noise_at = 8, 3
    frames = _sequence(n, noise_at)
    try:
        free = list(FrameRunner(ctx, 3, (240, 320), track=True, detect="slots").stream(frames))
        _check_slots_policy(free, None, None, 1.5)
        sc = np.array([r["track_score"] for r in free])
        others = np.delete(sc.reshape(-1), noise_at * 3)
        assert sc[noise_at, 0] < others.min(), "the faint frame is meant to score lowest"
        min_score = float((sc[noise_at, 0] + others.min()) / 2)
        res = list(FrameRunner(ctx, 3, (240, 320), track=True, detect="slots", min_score=min_score).stream(frames))
        staggered = list(FrameRunner(ctx, 3, (240, 320), track=True, detect="slots", redetect_every=2).stream(frames))
    finally:
        ctx.release_graphs()
    _check_slots_policy(res, None, min_score, 1.5)
    det = np.array([r["track_detected"] for r in res])
    want = np.zeros_like(det)
    want[0] = True
    want[noise_at + 1, 0] = True                   # lost at t -> re-detected at t + 1, that slot only
    np.testing.assert_array_equal(det, want)
    _check_slots_policy(staggered, 2, None, 1.5)
    sdet = np.array([r["track_detected"] for r in staggered])
    assert all(sdet[t][S.redetect_force(3, 2, t) != 0].all() for t in range(n))   # every forced slot re-detects
    # eager against graph replay: the same steps, enqueued one by one
    st = runtime.TrackState(3)
    hs = _dev(np.array([[1.0, 0.0]] * 3, F))
    for t, f in enumerate(frames):
        image = ctx.resize_frames(_dev(f), 240, 320, normalize=True)
        r = _host(ctx.track_step_slots(image, hs, st, margin=1.5, min_score=min_score, outputs="keypoints"))
        for k in ("keypoints_uv", "keypoint_coord3d", "center", "scale_crop", "track_detected"):
            _bits_equal(r[k], res[t][k], "%s at step %d" % (k, t))


def test_frame_runner_slots_submit_does_not_synchronise(ctx):
    ctx.set_precision("bf16x3")
    frames = [torch.from_numpy(f).cuda() for f in _sequence(4, noise_at=2)]
    try:
        runner = FrameRunner(ctx, 3, (240, 320), track=True, detect="slots", redetect_every=3, min_score=0.0)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            outs = [runner.submit(f) for f in frames]
        finally:
            torch.cuda.set_sync_debug_mode("default")
        torch.cuda.synchronize()
        assert "detected" not in outs[0] and outs[-1]["track_detected"].shape == (3,)
    finally:
        ctx.release_graphs()
    with pytest.raises(ValueError):
        FrameRunner(ctx, 3, (240, 320), track=True, detect="every")
    with pytest.raises(ValueError):
        FrameRunner(ctx, 3, (240, 320), detect="slots")         # per-slot re-detection needs tracking


def _kernels(fn):
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def test_bad_arguments_are_refused_before_any_launch(ctx):
    ctx.set_precision("bf16x3")
    B, H, W = 1, 240, 320
    img = torch.zeros((B, H, W, 3), dtype=torch.float32, device="cuda")
    big = torch.zeros((1, 2049, 64, 3), dtype=torch.float32, device="cuda")
    hs = torch.zeros((B, 2), dtype=torch.float32, device="cuda")
    c3d = torch.zeros((B, 21, 3), dtype=torch.float32, device="cuda")
    st = runtime.TrackState(B)
    P = _lib.C.c_void_p
    nan = float("nan")

    def step(image=img, b=B, h=H, w=W, margin=1.5, min_score=nan, state=st.buffer, pose3d=1, coord=c3d):
        return ctx.lib.h3d_track_step_slots(ctx.h, P(image.data_ptr()), P(hs.data_ptr()), b, h, w, pose3d, margin, min_score,
                                            None if state is None else P(state.data_ptr()), None, None, None, None, None, None,
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
    with pytest.raises(ValueError):
        ctx.track_step_slots(img, hs, st, force=torch.zeros(B + 1, dtype=torch.int32, device="cuda"))

"""Cases and delay patterns of tests/test_gpu_schedule_skew.py, and the child process that runs them on the schedule-skew library.

The skew variant (python -m hand3d_b200.build --skew) is the product library with the H3D_SKEW hooks of csrc/skew.cuh compiled in: a
hook sleeps at an existing synchronisation point when the skew_* tuning keys ask it to.  It is only ever loaded in a child process
(`python tests/schedule_skew_cases.py OUT.npz`), which points _lib.LIB_PATH at it before the first load, runs every case under every
pattern and saves the outputs; the test process runs the same cases on the product library and compares them bit for bit.

A case is run(ctx) -> {name: numpy array}; check(out) (optional) holds the outputs against the existing reference at the existing bound,
reusing the problems, references and bounds of the suite's own tests."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

# skew.cuh: sites and roles
SITES = ("producer", "consumer", "commit", "epilogue", "cluster", "pdl_tail", "ticket")
ALL, WG0, WG1, WG2, EVEN_CTA, ODD_CTA, LAST_RANK, RANK0 = 0, 1, 2, 3, 4, 5, 6, 8
MAX_NS = 4000


def _site(site, ns, role=ALL, period=0, seed=0):
    return [("skew_%s_ns" % site, ns), ("skew_%s_role" % site, role), ("skew_%s_period" % site, period), ("skew_%s_seed" % site, seed)]


def _mix(seed):
    """Every site delayed by a pseudo-random 0..3 us, hashed per (CTA, warpgroup, site, iteration)."""
    return [kv for i, s in enumerate(SITES) for kv in _site(s, 3000, seed=seed * 7919 + i + 1)]


# pattern name -> h3d_set_tuning (key, value) pairs applied after skew_reset
PATTERNS = {
    "none": [],
    "producer_slow": _site("producer", 2000, WG0),
    "wg1_slow": _site("consumer", 2000, WG1),
    # conv_wgrad: warpgroup 1 runs a whole ring ahead of warpgroup 2, the schedule of the odd-ring race
    "wg2_slow": _site("consumer", 2000, WG2),
    "commit_wait_wide": _site("commit", 2000),
    "epilogue_wg1_slow": _site("epilogue", 3000, WG1),
    "cluster_rank0_slow": _site("cluster", 3000, RANK0 + 0) + _site("ticket", 3000, RANK0 + 0),
    "cluster_last_slow": _site("cluster", 3000, LAST_RANK) + _site("ticket", 3000, LAST_RANK),
    # the dependent grid starts (griddepcontrol.launch_dependents) against a primary that then waits before storing anything
    "pdl_tail_slow": _site("pdl_tail", MAX_NS) + _site("epilogue", 1000, ALL, period=2),
    # the same with the odd CTAs only: a primary whose CTAs store at different times, its dependents resident on the SMs it vacates
    "pdl_tail_odd_slow": _site("pdl_tail", MAX_NS, ODD_CTA) + _site("epilogue", MAX_NS, ODD_CTA),
    "random_1": _mix(1),
    "random_2": _mix(2),
    "random_3": _mix(3),
}


def apply_pattern(ctx, name):
    ctx.set_tuning("skew_reset", 1)
    for k, v in PATTERNS[name]:
        ctx.set_tuning(k, v)


# ---------------------------------------------------------------------------------------------------------------- cases
def _cu(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _np(t):
    return t.detach().cpu().numpy()


# conv_tc_kernel: all nine instances on one 1x1 layer, 2 x 128 x 128, Cin 320 -> Cout 128.  256 pixel tiles (512 at N = 64) on at most
# 132 persistent CTAs: two to four tiles per CTA.  5 K blocks per tile is not a multiple of any ring (3 stages at <128,3>, 4 at <64,3>
# and <64,4>, 6 at <128,1>, 8 at <64,1>), so the ring phase wraps inside a tile.
CONV_SHAPE = (2, 128, 128, 320, 128, 1, 1)
CONV_INST = [(bn, prec) for bn in (64, 128) for prec in ("bf16x3", "fp16x3", "bf16", "fp16")] + [(64, "fp16_f8c")]


def _conv_tc(bn, prec):
    def run(ctx):
        import test_gpu_conv_tiles as T
        x, w, b, _ = T.fwd_problem(*CONV_SHAPE)
        ctx.set_tuning("tc_bn", bn)
        try:
            if prec == "fp16_f8c":   # its scales come from host weights
                out = {"y": _np(ctx.conv2d_tc(_cu(x), w, b, leaky=True, precision=prec))}
            else:
                out = {"y": _np(ctx.conv2d_tc_dev(_cu(x), _cu(w), _cu(b), leaky=True, precision=prec))}
            if prec in ("bf16x3", "bf16"):   # the integer canary is stated for bf16 planes
                xi, wi, bi = T.int_problem(*CONV_SHAPE[:6], prec)
                out["canary"] = T.conv_guarded(ctx, xi, wi, bi, prec=prec)
        finally:
            ctx.set_tuning("tc_bn", 0)
        return out

    def check(out):
        import test_gpu_conv_tiles as T
        from oracle import tf1_ops
        x, w, b, ref = T.fwd_problem(*CONV_SHAPE)
        err = np.abs(out["y"] - tf1_ops.leaky_relu(ref)).max()
        assert err < T.TOL[prec], "max abs err %.3e (tolerance %.1e)" % (err, T.TOL[prec])
        if "canary" in out:
            xi, wi, bi = T.int_problem(*CONV_SHAPE[:6], prec)
            T.assert_exact(out["canary"], T.int_reference(xi, wi, bi, 1), "integer canary")
    return run, check


def _conv_shape(shape, prec):
    """A shape of test_gpu_conv_tiles.py against its fp64 reference: stride 2, or a K-block count past a fold of the partial sum."""
    def run(ctx):
        import test_gpu_conv_tiles as T
        x, w, b, _ = T.fwd_problem(*shape)
        return {"y": _np(ctx.conv2d_tc_dev(_cu(x), _cu(w), _cu(b), stride=shape[6], leaky=True, precision=prec))}

    def check(out):
        import test_gpu_conv_tiles as T
        from oracle import tf1_ops
        err = np.abs(out["y"] - tf1_ops.leaky_relu(T.fwd_problem(*shape)[3])).max()
        assert err < T.TOL[prec], "max abs err %.3e (tolerance %.1e)" % (err, T.TOL[prec])
    return run, check


# conv_wgrad_tc_kernel <BN, PASSES>: BN = 128 where Cin % 128 == 0, 3 passes in bf16x3 and 1 in bf16.  Shapes of test_gpu_conv_tiles.py's
# BWD_SHAPES: 600 (here 800) CTA tiles leave no room for a split; a 41 x 45 map shares 72 pixel blocks among many splits.
WGRAD = {"nosplit": {64: (2, 9, 7, 192, 512, 5, 1), 128: (2, 9, 7, 256, 512, 5, 1)},
         "split": {64: (2, 41, 45, 64, 64, 3, 1), 128: (2, 41, 45, 128, 64, 3, 1)}}


def _wgrad(shape, prec, check_ref=True):
    def run(ctx):
        import test_gpu_conv_backward as B
        x, w, b, dy = B._problem(shape)
        xg, wg, bg, dyg = _cu(x), _cu(w), _cu(b), _cu(dy)
        y = ctx.conv2d_tc_dev(xg, wg, bg, stride=shape[6], leaky=True, precision=prec)
        dx, dw, db = ctx.conv2d_tc_backward(xg, y, dyg, wg, stride=shape[6], leaky=True, precision=prec, need_dx=check_ref,
                                             need_db=check_ref)
        out = {"y": _np(y), "dw": _np(dw)}
        if check_ref:
            out.update(dx=_np(dx), db=_np(db))
        return out

    def check(out):
        import test_gpu_conv_backward as B
        from oracle import tf1_grads as G
        x, w, b, dy = B._problem(shape)
        rdx, rdw, rdb = G.conv_grads(x, w, b, dy, shape[6], leaky=True, pre=out["y"])
        for name, g, r in (("dx", out["dx"], rdx), ("dw", out["dw"], rdw), ("db", out["db"], rdb)):
            e = B._err(g, r)
            assert e < B.TOL[prec][name], "%s normwise error %.3e (bound %.1e)" % (name, e, B.TOL[prec][name])
    return run, (check if check_ref else None)


# fc_chain_kernel: the lifting stage (PosePrior and ViewpointNet chains, so the rotation epilogue's ticket is taken)
def _lifting(B, prec):
    def _ctx_weights(ctx):
        import test_gpu_lifting as L
        if not getattr(ctx, "_skew_lift_weights", False):
            ctx.load_weights(L.W_STD)
            ctx._skew_lift_weights = True
        return L

    def run(ctx):
        L = _ctx_weights(ctx)
        ctx.set_precision(prec)
        try:
            out, can, rot = ctx.lifting(_cu(L.SM[:B]), _cu(L.HS[:B]), "proposed")
            return {"out": _np(out), "can": _np(can), "rot": _np(rot)}
        finally:
            ctx.set_precision("bf16x3")

    def check(out):
        import test_gpu_lifting as L
        ref = dict(zip(("out", "can", "rot"), L.oracle("proposed")))
        for k in ("out", "can", "rot"):
            e = float(np.abs(out[k].astype(np.float64) - ref[k][:B]).max() / np.abs(ref[k][:B]).max())
            bound = L.BOUND["chain_" + prec][k]
            assert e < bound, "%s normwise error %.3e (bound %.1e)" % (k, e, bound)
    return run, check


# mask_grow_cluster_kernel (sides > 512: a cluster per image, 8 CTAs at 2048 rows) and the single-CTA grower, against grow_oracle.py
def _grow(H, W):
    def _logits():
        import grow_oracle as G
        kinds = G.KINDS if H * W <= 600 * 800 else G.KINDS[:1]
        return G.logits_of([G.make_case(H, W, k, seed=H + W + i) for i, k in enumerate(kinds)])

    def run(ctx):
        r = ctx.seg_postprocess(_cu(_logits()))
        return {k: _np(v) for k, v in r.items()}

    def check(out):
        import grow_oracle as G
        ref = G.seg_postprocess(_logits())
        for k in ("hand_mask", "max_loc", "center", "crop_size", "scale_crop"):
            assert np.array_equal(out[k].reshape(ref[k].shape), ref[k]), k
    return run, check


# the whole pipeline at B = 2, 320 x 320: conv_c3_tc_kernel, conv_tc_kernel with fused pools and strides behind PDL, seg_prob, the
# growers, the key-point arg-max and fc_chain_kernel.  The suite's pipeline tests hold these outputs against the oracle; here they
# must not move by a bit under any schedule.
def _pipeline(prec):
    def run(ctx):
        from hand3d_b200 import weights as Wt
        if not getattr(ctx, "_skew_pipe_weights", False):
            ctx.load_weights(Wt.synthetic_weights(0))
            ctx._skew_pipe_weights = True
            ctx._skew_lift_weights = False
        ctx.set_precision(prec)
        try:
            img = Wt.synthetic_images(2, 320, 320, seed=5)
            hs = np.array([[1.0, 0.0], [0.0, 1.0]], np.float32)
            r = ctx.pipeline(_cu(img), _cu(hs), want_mask=True)
            return {k: _np(v) for k, v in r.items() if v is not None}
        finally:
            ctx.set_precision("bf16x3")
    return run, None


# first-occurrence arg-max keys (heatmap_argmax_kernel, resize_argmax(_pow2)_kernel): every channel's maximum planted twice or more
def _planted_maxima(B, H, W):
    rng = np.random.default_rng(808)
    sm = rng.uniform(-1, 1, size=(B, H, W, 21)).astype(np.float32)
    for b in range(B):
        for c in range(21):
            for _ in range(1 + c % 3):
                sm[b, rng.integers(0, H), rng.integers(0, W), c] = 5.0
            sm[b, H - 1, W - 1, c] = 5.0    # a tie at the very last pixel, read by the last CTA
    return sm


def _detect():
    def run(ctx):
        return {"uv": _np(ctx.detect_keypoints(_cu(_planted_maxima(3, 256, 256))))}

    def check(out):
        from oracle import hand3d_oracle as O
        sm = _planted_maxima(3, 256, 256)
        for b in range(3):
            assert np.array_equal(out["uv"][b], O.detect_keypoints(sm[b]).astype(np.int32)), b
    return run, check


def _upsample_detect(out_hw):
    def run(ctx):
        up, uv = ctx.upsample_detect_keypoints(_cu(_planted_maxima(2, 32, 32)), out_hw, out_hw)
        return {"up": _np(up), "uv": _np(uv)}

    def check(out):
        # uv against the first-occurrence arg-max of the kernel's own up-sampled maps: the ties are what this checks.  The maps
        # themselves are held to the product library bit for bit here, and to the resize oracle by test_gpu_ops.py.
        from oracle import hand3d_oracle as O
        for b in range(2):
            assert np.array_equal(out["uv"][b], O.detect_keypoints(out["up"][b]).astype(np.int32)), b
    return run, check


# counted batches: a slots step (h3d_track_step_slots) with slots 0 and 2 of 4 lost runs HandSegNet on a device-counted batch of 2,
# conv_c3_tc_kernel<COUNTED> reading the selected slots in place and every conv_tc_kernel layer with its count.
# test_gpu_track_slots.py holds these outputs to a detect step for the selected slots and a track step for the others.
_TRACK = {}


def _track_slots(prec):
    def run(ctx):
        import torch
        from hand3d_b200 import runtime
        from hand3d_b200 import weights as Wt
        if "ctx" not in _TRACK:
            _TRACK["ctx"] = runtime.Context()
            _TRACK["ctx"].load_weights(Wt.synthetic_weights(0, seg_shift=0.15))
        tc = _TRACK["ctx"]
        tc.set_precision(prec)
        st = runtime.TrackState(4)
        st.lost.copy_(torch.tensor([1, 0, 1, 0], dtype=torch.int32))
        img = Wt.synthetic_images(4, 240, 320, seed=11)
        hs = np.eye(2, dtype=np.float32)[[0, 1, 1, 0]]
        r = tc.track_step_slots(_cu(img), _cu(hs), st)
        out = {k: _np(v) for k, v in r.items() if v is not None}
        out["state"] = _np(st.buffer)
        return out
    return run, None


# one training step of each network at B = 2, 64 x 64 (test_gpu_training.py's batches): forward, loss, backward and Adam, whose
# ticket (adam_step_kernel) advances the bias corrections.  test_gpu_training.py holds these steps to fp64.
_NET = {}


def _train_step(scope):
    def run(ctx):
        import torch
        import test_gpu_training as Tr
        from hand3d_b200 import runtime
        from hand3d_b200 import weights as Wt
        from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork
        dctx = runtime.default_context()
        dctx.set_precision("bf16x3")
        if "net" not in _NET:
            _NET["net"] = ColorHandPose3DNetwork()
            _NET["net"].init(weights=Wt.synthetic_weights(0))
        net = _NET["net"]
        batch = [Tr._cu(a) for a in (Tr._pose_batch(27) if scope == "PoseNet2D" else Tr._seg_batch(27))]
        v, opt = Tr._fresh(dctx, scope)
        opt.zero_grad()
        loss = Tr._pose_loss(net, *batch)[0] if scope == "PoseNet2D" else Tr._seg_loss(net, *batch)[0]
        loss.backward()
        opt.step()
        torch.cuda.synchronize()
        out = {"loss": _np(loss).reshape(1)}
        out.update({n.replace("/", "."): _np(p) for n, p in v.items()})
        return out
    return run, None


CASES = {}
for _bn, _prec in CONV_INST:
    CASES["conv_tc_%d_%s" % (_bn, _prec)] = _conv_tc(_bn, _prec)
CASES["conv_tc_stride2"] = _conv_shape((3, 10, 18, 192, 128, 7, 2), "bf16x3")
CASES["conv_tc_fold"] = _conv_shape((2, 9, 13, 1216, 64, 1, 1), "fp16x3")
for _split, _shapes in WGRAD.items():
    for _bn, _shape in _shapes.items():
        for _prec in ("bf16x3", "bf16"):
            CASES["wgrad_%d_%s_%s" % (_bn, _split, _prec)] = _wgrad(_shape, _prec)
CASES["wgrad_conv1_2_8x256x256"] = _wgrad((8, 256, 256, 64, 64, 3, 1), "bf16x3", check_ref=False)
for _B in (13, 129):
    for _prec in ("bf16x3", "fp16x3"):
        CASES["fc_chain_B%d_%s" % (_B, _prec)] = _lifting(_B, _prec)
CASES["grow_cluster_600x800"] = _grow(600, 800)
CASES["grow_cluster_2048x2048"] = _grow(2048, 2048)
CASES["grow_single_320x320"] = _grow(320, 320)
CASES["pipeline_bf16x3"] = _pipeline("bf16x3")
CASES["pipeline_fp16x3"] = _pipeline("fp16x3")
CASES["detect_keypoints_ties"] = _detect()
CASES["upsample_detect_keypoints_ties"] = _upsample_detect(256)            # x8: resize_argmax_pow2_kernel
CASES["upsample_detect_keypoints_ties_240"] = _upsample_detect(240)        # 7.5x: resize_argmax_kernel
CASES["track_slots_counted_bf16x3"] = _track_slots("bf16x3")
CASES["track_slots_counted_fp16x3"] = _track_slots("fp16x3")
CASES["train_step_PoseNet2D"] = _train_step("PoseNet2D")
CASES["train_step_HandSegNet"] = _train_step("HandSegNet")


def run_cases(ctx, patterns=None):
    """{(pattern, case): outputs}.  Without patterns: the cases once, as the library runs them unconfigured."""
    import torch
    out = {}
    for pat in (patterns or [None]):
        if pat is not None:
            apply_pattern(ctx, pat)
        for name, (run, _) in CASES.items():
            out[(pat, name)] = run(ctx)
            torch.cuda.synchronize()
        ctx.check_errors()
    if patterns:
        ctx.set_tuning("skew_reset", 1)
    return out


def main(path):
    """Child process: build and load the skew library, run every case under every pattern, save the outputs to `path`."""
    from hand3d_b200 import _lib, build
    _lib.LIB_PATH = build.build(skew=True)
    from hand3d_b200 import runtime
    ctx = runtime.Context()
    res = run_cases(ctx, list(PATTERNS))
    np.savez(path, **{"%s/%s/%s" % (p, c, k): v for (p, c), d in res.items() for k, v in d.items()})
    print("schedule skew: %d patterns x %d cases" % (len(PATTERNS), len(CASES)))


if __name__ == "__main__":
    main(sys.argv[1])

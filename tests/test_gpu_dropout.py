"""Dropout of the lifting stage on the GPU (csrc/dropout.cu, h3d_set_dropout, evaluation=False): the kernels against the numpy
restatement (tests/dropout_oracle.py) bit for bit, the lifting with dropout against an fp64 restatement that uses the device's keep
bits, whole-network training gradients, training runs, CUDA-graph replay, the pipeline and the track step, the default (disabled)
behaviour, refused arguments and poisoned scratch.

The module runs on a context of its own, installed as the default for its duration: the seed it sets and the weights it loads do not
reach other test modules."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

import dropout_oracle as D
import lift_train_oracle as L
import test_gpu_lifting_training as LT
from hand3d_b200 import _lib
from hand3d_b200 import weights as Wt
from oracle import hand3d_oracle as O

pytestmark = pytest.mark.gpu
f32, f64 = np.float32, np.float64
KEEP = {"fc_rel0": (0.8, 0), "fc_rel1": (0.8, 1), "fc_vp0": (0.75, 2), "fc_vp1": (0.75, 3)}
VARIANTS = ["direct", "bottleneck", "local", "proposed"]
PRECISIONS = ["bf16x3", "fp16x3", "bf16", "fp16", "fp32_ffma", "fp16_f8c"]
# tests/test_gpu_lifting.py's bounds of the two routes the dropout plan takes: the layer-by-layer tensor-core route (fc_chain = 0) and
# the fp32 CUDA-core route (fp32_ffma, fp16_f8c)
BOUND_TC = {"out": 1.8e-4, "can": 8.2e-5, "rot": 1.5e-4}
BOUND_F32 = {"out": 1.2e-5, "can": 4.1e-6, "rot": 1.5e-5}
W_STD = {k: v for k, v in Wt.synthetic_weights(0).items() if k.startswith(("PosePrior", "ViewpointNet"))}
W_BOTT = {k: v for k, v in Wt.synthetic_weights(0, bottleneck=True).items() if k.startswith("PosePrior")}


@pytest.fixture(scope="module")
def ctx():
    from hand3d_b200 import runtime
    saved = dict(runtime._default)
    runtime._default.clear()
    c = runtime.default_context()
    c.set_precision("bf16x3")
    c.set_dropout(1234)
    yield c
    torch.cuda.synchronize()
    c.set_dropout(None)
    runtime._default.clear()
    runtime._default.update(saved)
    del c
    gc.collect()
    torch.cuda.empty_cache()


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _np(t):
    return t.detach().cpu().numpy()


def _draw(ctx):
    return int(ctx.dropout_state().item())


def _s():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


# ---------------------------------------------------------------------------------------------------- 1. the kernels, bit for bit
@pytest.mark.parametrize("keep_prob", [0.8, 0.75, 0.5])
@pytest.mark.parametrize("cols", [128, 256, 512, 37])
@pytest.mark.parametrize("rows", [1, 8, 129, 160])
def test_kernels_vs_oracle(ctx, rows, cols, keep_prob):
    rng = np.random.default_rng(rows * 1000 + cols)
    x = (rng.normal(size=(rows, cols)) * rng.choice([1e-3, 1.0, 1e4], size=(rows, cols))).astype(f32)
    dy = rng.normal(size=(rows, cols)).astype(f32)
    xd, dyd = _cu(x), _cu(dy)
    stride = (cols + 63) // 64 * 64
    seen = []
    for seed, draw in ((1234, 0), (1234, 5), (99, 5)):
        ctx.set_dropout(seed)
        ctx.load_dropout_state(draw)
        for half in (0, 1):
            y = torch.full((rows, cols), float("nan"), device="cuda")
            keep = torch.full((rows, cols), 7, dtype=torch.uint8, device="cuda")
            hi = torch.full((rows, stride), 0x7FFF, dtype=torch.int16, device="cuda")
            lo = torch.full((rows, stride), 0x7FFF, dtype=torch.int16, device="cuda")
            _lib.check(ctx.lib.h3d_dropout_forward_planes(ctx.h, _p(xd), rows, cols, keep_prob, 2, _p(y), _p(keep), half, stride, _p(hi),
                                                          _p(lo), _s()), "h3d_dropout_forward_planes")
            y_ref, k_ref = D.dropout(x, seed, draw, 2, keep_prob)
            assert np.array_equal(_np(keep), k_ref)
            assert np.array_equal(_np(y).view(np.uint32), y_ref.view(np.uint32))
            hi_ref, lo_ref = D.planes(y_ref, stride, half)
            assert np.array_equal(_np(hi).view(np.uint16), hi_ref)
            assert np.array_equal(_np(lo).view(np.uint16), lo_ref)
        y2, k2 = ctx.dropout_forward(xd, keep_prob, 2)                   # the plain entry: the same draw gives the same result
        assert torch.equal(k2, keep) and torch.equal(y2, y)
        dx = ctx.dropout_backward(dyd, k2, keep_prob)
        dx_ref = D.backward(dy, (k_ref.astype(f32), keep_prob))
        assert np.array_equal(_np(dx).view(np.uint32), dx_ref.view(np.uint32))
        assert _draw(ctx) == draw                                         # the kernels read the draw, they do not advance it
        seen.append(_np(keep))
    if rows * cols >= 128:                                                # another draw or seed: other masks
        assert not np.array_equal(seen[0], seen[1]) and not np.array_equal(seen[1], seen[2])
    ctx.dropout_advance()
    assert _draw(ctx) == 6
    ctx.set_dropout(1234)


def test_in_place_and_keep_prob_one(ctx):
    x = _cu(np.random.default_rng(5).normal(size=(8, 512)).astype(f32))
    ctx.load_dropout_state(3)
    y, k = ctx.dropout_forward(x, 0.8, 0)
    z = x.clone()
    _lib.check(ctx.lib.h3d_dropout_forward(ctx.h, _p(z), 8, 512, C.c_float(0.8), 0, _p(z), None, _s()), "in place")
    assert torch.equal(z, y)
    y1, k1 = ctx.dropout_forward(x, 1.0, 0)
    assert torch.equal(y1, x) and bool((k1 == 1).all())
    ctx.set_dropout(1234)


# ---------------------------------------------------------------------------------------------------- 2. lifting inference
def _masks(ctx, draw, B, layers):
    """Keep bits (fp64 [B, cols] / keep_prob) of the lifting's dropout layers at `draw`, from the standalone kernel."""
    saved = ctx.dropout_state()
    ctx.load_dropout_state(draw)
    out = {}
    for name in layers:
        kp, layer = KEEP[name]
        cols = {"fc_rel0": 512, "fc_rel1": 512, "fc_vp0": 256, "fc_vp1": 128}[name]
        _, k = ctx.dropout_forward(torch.ones((B, cols), device="cuda"), kp, layer)
        out[name] = _np(k).astype(f64) / kp
    ctx.load_dropout_state(saved)
    return out


def _fc(x, wd, scope, name, relu, m=None):
    y = x @ wd["%s/%s/weights" % (scope, name)].astype(f64) + wd["%s/%s/biases" % (scope, name)].astype(f64)
    if relu:
        y = np.maximum(y, 0.01 * y)
    return y * m[name] if m is not None and name in m else y


def _ref_lifting(sm, hs, wd, variant, m):
    """fp64 lifting (oracle/hand3d_oracle.py's layers) with the dropout masks m applied after the hidden FC layers."""
    def branch(scope, convs, fcs):
        x = sm.astype(f64)
        for i in range(3):
            x = O._conv(x, wd, scope, convs % (i, 1), 1, dtype=f64)
            x = O._conv(x, wd, scope, convs % (i, 2), 2, dtype=f64)
        x = np.concatenate([x.reshape(len(x), -1), hs.astype(f64)], 1)
        for n in fcs:
            x = _fc(x, wd, scope, n, True, m)
        return x
    x = branch("PosePrior", "conv_pose_%d_%d", ["fc_rel0", "fc_rel1"])
    if variant == "bottleneck":
        x = _fc(x, wd, "PosePrior", "fc_bottleneck", False)
    can = _fc(x, wd, "PosePrior", "fc_xyz", False).reshape(-1, 21, 3)
    if variant == "local":
        return O.bone_rel_trafo_inv(can), can, None
    if variant != "proposed":
        return can, can, None
    v = branch("ViewpointNet", "conv_vp_%d_%d", ["fc_vp0", "fc_vp1"])
    u = np.concatenate([_fc(v, wd, "ViewpointNet", "fc_vp_u%s" % a, False) for a in "xyz"], 1)
    R, out = L.rotate_canonical(can, u, hs)
    return out, can, R


def _lift_inputs(B, seed=7):
    rng = np.random.default_rng(seed)
    sm = rng.normal(size=(B, 32, 32, 21)).astype(f32)
    hs = np.zeros((B, 2), f32)
    hs[np.arange(B), rng.integers(0, 2, B)] = 1
    return sm, hs


def _err(g, ref):
    return float(np.abs(_np(g).astype(f64) - ref).max() / np.abs(ref).max())


@pytest.mark.parametrize("prec", PRECISIONS)
@pytest.mark.parametrize("variant", VARIANTS)
def test_lifting_with_dropout_vs_fp64(ctx, variant, prec):
    B = 13
    wd = W_BOTT if variant == "bottleneck" else W_STD
    ctx.load_weights(wd)
    ctx.set_precision(prec)
    try:
        sm, hs = _lift_inputs(B)
        ctx.load_dropout_state(4)
        got = ctx.lifting(_cu(sm), _cu(hs), variant, dropout=True)
        assert _draw(ctx) == 5                                            # one forward is one draw
        layers = ["fc_rel0", "fc_rel1"] + (["fc_vp0", "fc_vp1"] if variant == "proposed" else [])
        ref = _ref_lifting(sm, hs, wd, variant, _masks(ctx, 4, B, layers))
        bound = BOUND_F32 if prec in ("fp32_ffma", "fp16_f8c") else BOUND_TC
        for k, g, r in zip(("out", "can", "rot"), got, ref):
            if r is not None:
                e = _err(g, r)
                assert e < bound[k], (k, e)
        other = _ref_lifting(sm, hs, wd, variant, _masks(ctx, 5, B, layers))   # the masks of another draw do not fit
        assert _err(got[1], other[1]) > 100 * bound["can"]
        ctx.load_dropout_state(4)
        again = ctx.lifting(_cu(sm), _cu(hs), variant, dropout=True)
        for a, b in zip(got, again):
            assert (a is None and b is None) or torch.equal(a, b)
    finally:
        ctx.set_precision("bf16x3")


# ---------------------------------------------------------------------------------------------------- 3. training
def _ref_branch(pooled, hs, v, scope, layers, fcs, heads, dec, m):
    from hand3d_b200 import arch  # noqa: F401
    x = pooled
    for name, k, stride, _, _, leaky in layers:
        x = LT._ref_conv(x, v["%s/%s/weights" % (scope, name)], v["%s/%s/biases" % (scope, name)], stride, leaky, dec)
    x = torch.cat([x.reshape(x.shape[0], -1), hs], 1)
    for name in fcs:
        x = LT._ref_fc(x, v["%s/%s/weights" % (scope, name)], v["%s/%s/biases" % (scope, name)], True, dec) * m.pop(0)
    for ws, bs in heads:
        x = LT._ref_fc(x, ws(v), bs(v), False, dec)
    return x


class _Keeps:
    """Records the keep bits (/ keep_prob) of every autograd.dropout call, as the fp64 reference forces them."""

    def __init__(self, monkeypatch, ctx):
        from hand3d_b200 import autograd as A
        self.m = []
        orig = A.dropout

        def rec(x, keep_prob, layer):
            y = orig(x, keep_prob, layer)
            _, k = ctx.dropout_forward(x.detach(), keep_prob, layer)
            self.m.append(k.cpu().double() / keep_prob)
            return y

        monkeypatch.setattr(A, "dropout", rec)


@pytest.mark.parametrize("variant", ["direct", "bottleneck", "local", "local_w_xyz_loss", "proposed"])
def test_whole_network_gradients_with_dropout_vs_fp64(ctx, variant, monkeypatch):
    from hand3d_b200 import arch
    from hand3d_b200.nets.PosePriorNetwork import PosePriorNetwork
    LT._load(ctx, variant)
    v = {}
    for s in LT._scopes(variant):
        v.update(ctx.variables(s))
    for p in v.values():
        p.grad = None
    sm, t = LT._batch(41)
    dec = LT._Decisions(monkeypatch)
    keeps = _Keeps(monkeypatch, ctx)
    d0 = _draw(ctx)
    _, coord3d, R = PosePriorNetwork(variant).inference(sm, t["hand_side"], evaluation=False, train=True)
    assert _draw(ctx) == d0 + 1
    loss = LT._loss(variant, coord3d, R, t)
    loss.backward()
    loss = float(loss.detach())
    assert len(keeps.m) == (4 if variant == "proposed" else 2)
    assert all(float((k == 0).float().mean()) > 0.05 for k in keeps.m)
    pooled = ctx.avg_pool8(sm).cpu().double()
    rv = {k: torch.nn.Parameter(p.detach().cpu().double()) for k, p in v.items()}
    tc = {k: x.detach().cpu().double() for k, x in t.items()}
    pp = [(lambda v, n=n: v["PosePrior/%s/weights" % n], lambda v, n=n: v["PosePrior/%s/biases" % n])
          for n in (["fc_bottleneck"] if variant == "bottleneck" else []) + ["fc_xyz"]]
    m = list(keeps.m)
    c_ref = _ref_branch(pooled, tc["hand_side"], rv, "PosePrior", arch.POSEPRIOR[:6], ["fc_rel0", "fc_rel1"], pp, dec, m).reshape(-1, 21, 3)
    if variant in ("direct", "bottleneck"):
        ref = torch.mean((c_ref - tc["keypoint_xyz21_normed"]) ** 2)
    elif variant == "local":
        ref = torch.mean((c_ref - tc["keypoint_xyz21_local"]) ** 2)
    elif variant == "local_w_xyz_loss":
        ref = torch.mean((L.bone_rel_trafo_inv_torch(c_ref) - tc["keypoint_xyz21_normed"]) ** 2)
    else:
        heads = [(lambda v: torch.cat([v["ViewpointNet/fc_vp_u%s/weights" % a] for a in "xyz"], 1),
                  lambda v: torch.cat([v["ViewpointNet/fc_vp_u%s/biases" % a] for a in "xyz"], 0))]
        u = _ref_branch(pooled, tc["hand_side"], rv, "ViewpointNet", arch.VIEWPOINT[:6], ["fc_vp0", "fc_vp1"], heads, dec, m)
        R_ref, _ = L.rotate_canonical_torch(c_ref, u, tc["hand_side"])
        ref = torch.mean((c_ref - tc["keypoint_xyz21_can"]) ** 2) + torch.mean((R_ref - tc["rot_mat"]) ** 2)
    assert not dec.out and not m
    ref.backward()
    assert abs(loss - ref.item()) <= 1e-4 * abs(ref.item()), (loss, ref.item())
    worst = 0.0
    for k, p in v.items():
        assert p.grad is not None and p.grad.abs().max().item() > 0, k
        e = LT._err(_np(p.grad), rv[k].grad.numpy())
        worst = max(worst, e)
        assert e <= LT.NET_TOL, (k, e)
    print("%s with dropout: loss %.6e, worst normwise gradient error %.2e" % (variant, loss, worst))


def _train(ctx, steps, batch, seed=77):
    from hand3d_b200.nets.PosePriorNetwork import PosePriorNetwork
    from hand3d_b200.optim import Adam
    LT._load(ctx, "proposed")
    ctx.set_dropout(seed)
    params = [p for s in LT._scopes("proposed") for p in ctx.variables(s).values()]
    opt = Adam(params, lr=1e-4)
    net = PosePriorNetwork("proposed")
    sm, t = batch
    losses = []
    for _ in range(steps):
        opt.zero_grad()
        _, coord3d, R = net.inference(sm, t["hand_side"], evaluation=False, train=True)
        loss = LT._loss("proposed", coord3d, R, t)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    return losses, [p.detach().clone() for p in params]


def test_training_with_dropout_lowers_the_loss_and_is_reproducible(ctx):
    batch = LT._batch(44)
    l1, w1 = _train(ctx, 30, batch)
    l2, w2 = _train(ctx, 30, batch)
    print("proposed with dropout: first %.5e last %.5e" % (l1[0], l1[-1]))
    assert np.mean(l1[-5:]) < np.mean(l1[:5])
    assert l1 == l2
    assert all(torch.equal(a, b) for a, b in zip(w1, w2))
    _, w3 = _train(ctx, 3, batch, seed=78)
    _, w4 = _train(ctx, 3, batch)
    assert not all(torch.equal(a, b) for a, b in zip(w3, w4))
    ctx.set_dropout(1234)


def test_cuda_graph_replay_with_dropout_equals_eager_steps(ctx):
    from hand3d_b200.nets.PosePriorNetwork import PosePriorNetwork
    from hand3d_b200.optim import Adam
    sm, t = LT._batch(45)
    net = PosePriorNetwork("proposed")
    probe = torch.ones((8, 512), device="cuda")
    k = 3

    def fresh():
        LT._load(ctx, "proposed")
        ctx.set_dropout(4321)
        params = [p for s in LT._scopes("proposed") for p in ctx.variables(s).values()]
        for p in params:
            p.grad = None
        return params, Adam(params, lr=1e-4)

    def step(opt):
        opt.zero_grad()
        _, coord3d, R = net.inference(sm, t["hand_side"], evaluation=False, train=True)
        loss = LT._loss("proposed", coord3d, R, t)
        loss.backward()
        opt.step()
        return ctx.dropout_forward(probe, 0.5, 4)[1]

    params, opt = fresh()
    for _ in range(2 + k):
        step(opt)
    eager = [p.detach().clone() for p in params]
    params, opt = fresh()
    gc.collect()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step(opt)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        kb = step(opt)
    assert _draw(ctx) == 2                              # capture ran nothing: the counter moves on replay
    masks = []
    for _ in range(k):
        g.replay()
        masks.append(kb.clone())
    torch.cuda.synchronize()
    assert _draw(ctx) == 2 + k
    for a, b in zip(params, eager):
        assert torch.equal(a.detach(), b)
    assert not torch.equal(masks[0], masks[1]) and not torch.equal(masks[1], masks[2])
    del g
    ctx.set_dropout(1234)


def test_network_entries_with_dropout(ctx):
    """Every place the reference takes `evaluation`: train=True and train=False agree at the same draw (one draw per call), and the
    ColorHandPose3DNetwork entries give PosePriorNetwork('proposed')'s outputs."""
    from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork
    from hand3d_b200.nets.PosePriorNetwork import PosePriorNetwork
    from hand3d_b200.utils.general import NetworkOps
    LT._load(ctx, "proposed", seed=2)
    ctx.commit_variables("PosePrior")
    ctx.commit_variables("ViewpointNet")
    sm, t = LT._batch(43)
    pooled = ctx.avg_pool8(sm)
    hs = t["hand_side"]
    net = ColorHandPose3DNetwork()
    ev = torch.tensor(False)
    for train in (True, False):
        with torch.no_grad():
            ctx.load_dropout_state(9)
            out, can, R = PosePriorNetwork("proposed").inference(sm, hs, evaluation=ev, train=train)
            for fn, ref in ((net._inference_pose3d, out), (net._inference_pose3d_can, can), (net._inference_viewpoint, R)):
                ctx.load_dropout_state(9)
                got = fn(pooled, hs, evaluation=ev, train=train)
                assert torch.equal(got, ref), (fn.__name__, train)
                assert _draw(ctx) == 10
        if train:
            tr = (out, can, R)
    for a, b, tol in zip(tr, (out, can, R), (LT.LIFT_TOL["out"], LT.LIFT_TOL["can"], LT.LIFT_TOL["rot"])):
        assert LT._err(_np(a), _np(b).astype(f64)) <= tol
    ctx.load_dropout_state(2)
    x = torch.randn(4, 64, device="cuda")
    y = NetworkOps.dropout(x, 0.5, False)
    assert _draw(ctx) == 3 and torch.equal(y, ctx.dropout_forward(x, 0.5, _lib.DROPOUT_LAYER_OP)[0]) is False
    ctx.load_dropout_state(2)
    assert torch.equal(y, ctx.dropout_forward(x, 0.5, _lib.DROPOUT_LAYER_OP)[0])
    assert NetworkOps.dropout(x, 1.0, False) is x and NetworkOps.dropout(x, 0.5, True) is x


# ---------------------------------------------------------------------------------------------------- 4. pipeline and track step
def test_pipeline_and_track_step_with_dropout(ctx):
    from hand3d_b200.runtime import TrackState
    ctx.load_weights(Wt.synthetic_weights(0))
    B = 2
    img = _cu(Wt.synthetic_images(B, 240, 320, seed=3))
    hs = _cu(Wt.synthetic_hand_side(B, seed=4))
    off = ctx.pipeline(img, hs)
    ctx.load_dropout_state(6)
    on = ctx.pipeline(img, hs, dropout=True)
    assert _draw(ctx) == 7
    for k in off:
        if k == "keypoint_coord3d" or off[k] is None:
            continue
        assert torch.equal(off[k], on[k]), k
    assert not torch.equal(off["keypoint_coord3d"], on["keypoint_coord3d"])
    s2 = ctx.posenet(on["image_crop"])[2]
    ctx.load_dropout_state(6)
    lift = ctx.lifting(s2, hs, "proposed", dropout=True)[0]
    assert torch.equal(lift, on["keypoint_coord3d"])
    for step in ("track_step", "track_step_slots"):
        ctx.load_dropout_state(6)
        st = TrackState(B)
        r = ctx.track_step(img, hs, st, True, dropout=True) if step == "track_step" else ctx.track_step_slots(img, hs, st, dropout=True)
        assert torch.equal(r["keypoint_coord3d"], on["keypoint_coord3d"]), step
        assert _draw(ctx) == 7


# ---------------------------------------------------------------------------------------------------- 5. disabled, refused, poisoned
def test_disabled_is_bit_identical_to_a_context_that_never_enabled_it(ctx):
    from hand3d_b200 import runtime
    fresh = runtime.Context()
    try:
        for c in (ctx, fresh):
            c.load_weights(Wt.synthetic_weights(0))
        B = 2
        img = _cu(Wt.synthetic_images(B, 240, 320, seed=5))
        hs = _cu(Wt.synthetic_hand_side(B, seed=6))
        sm, hs13 = _lift_inputs(13)
        ctx.lifting(_cu(sm), _cu(hs13), "proposed", dropout=True)          # the switch was on just before
        for c in (ctx, fresh):
            c.set_precision("fp32_ffma")
        results = []
        for c in (ctx, fresh):
            r = [c.lifting(_cu(sm), _cu(hs13), v) for v in VARIANTS if v != "bottleneck"]
            c.set_precision("bf16x3")
            r += [c.lifting(_cu(sm), _cu(hs13), v) for v in VARIANTS if v != "bottleneck"]
            p = c.pipeline(img, hs)
            tr = c.track_step(img, hs, runtime.TrackState(B), True)
            results.append((r, p, tr))
        (ra, pa, ta), (rb, pb, tb) = results
        for x, y in zip(ra, rb):
            for a, b in zip(x, y):
                assert (a is None and b is None) or torch.equal(a, b)
        for k in pa:
            assert (pa[k] is None) == (pb[k] is None) and (pa[k] is None or torch.equal(pa[k], pb[k])), k
        for k in ta:
            assert (ta[k] is None) == (tb[k] is None) and (ta[k] is None or torch.equal(ta[k], tb[k])), k
        seed = ctx.dropout_seed
        ctx.set_dropout(None)
        with pytest.raises(NotImplementedError, match="set_dropout"):
            ctx.lifting(_cu(sm), _cu(hs13), "proposed", dropout=True)
        ctx.set_dropout(seed)
    finally:
        fresh.lib.h3d_destroy(fresh.h)
        fresh.h = None
        fresh._ws = None
        del fresh
        gc.collect()


def test_refused_arguments_enqueue_nothing(ctx):
    x = torch.ones((4, 8), device="cuda")
    y = torch.full((4, 8), 5.0, device="cuda")
    k = torch.full((4, 8), 9, dtype=torch.uint8, device="cuda")
    lib, h = ctx.lib, ctx.h
    torch.cuda.synchronize()
    n0, d0 = ctx.launch_count, _draw(ctx)
    ctx._dropout_mode(True)
    for kp in (0.0, -0.5, 1.5, float("nan"), float("inf")):
        assert lib.h3d_dropout_forward(h, _p(x), 4, 8, kp, 0, _p(y), _p(k), _s()) == _lib.EINVAL
        assert lib.h3d_dropout_backward(h, _p(x), _p(k), 4, 8, kp, _p(y), _s()) == _lib.EINVAL
    for rows, cols in ((0, 8), (4, 0), (-1, 8)):
        assert lib.h3d_dropout_forward(h, _p(x), rows, cols, 0.8, 0, _p(y), _p(k), _s()) == _lib.EINVAL
        assert lib.h3d_dropout_backward(h, _p(x), _p(k), rows, cols, 0.8, _p(y), _s()) == _lib.EINVAL
    assert lib.h3d_dropout_forward(h, _p(x), 4, 8, 0.8, -1, _p(y), _p(k), _s()) == _lib.EINVAL
    assert lib.h3d_dropout_forward_planes(h, _p(x), 4, 8, 0.8, 0, _p(y), _p(k), 0, 4, _p(k), None, _s()) == _lib.EINVAL
    assert lib.h3d_dropout_forward_planes(h, _p(x), 4, 8, 0.8, 0, _p(y), _p(k), 2, 8, _p(k), None, _s()) == _lib.EINVAL
    ctx._dropout_mode(False)
    assert lib.h3d_dropout_forward(h, _p(x), 4, 8, 0.8, 0, _p(y), _p(k), _s()) == _lib.EINVAL
    assert lib.h3d_dropout_backward(h, _p(x), _p(k), 4, 8, 0.8, _p(y), _s()) == _lib.EINVAL
    assert lib.h3d_dropout_advance(h, _s()) == _lib.EINVAL
    torch.cuda.synchronize()
    assert ctx.launch_count == n0 and _draw(ctx) == d0
    assert bool((y == 5.0).all()) and bool((k == 9).all())


@pytest.mark.parametrize("prec", ["bf16x3", "fp16x3", "fp32_ffma"])
def test_poisoned_scratch_changes_nothing(ctx, prec):
    ctx.load_weights(W_STD)
    ctx.set_precision(prec)
    try:
        sm, hs = _lift_inputs(13, seed=8)
        x = _cu(np.random.default_rng(9).normal(size=(13, 300)).astype(f32))
        runs = []
        for byte in (0, 0xFF, 0x7F):
            ctx.lifting(_cu(sm), _cu(hs), "proposed", dropout=True)         # sizes the workspace and builds the plan
            ctx.fill_scratch(byte)
            ctx.load_dropout_state(11)
            r = ctx.lifting(_cu(sm), _cu(hs), "proposed", dropout=True)
            ctx.load_dropout_state(11)
            y, k = ctx.dropout_forward(x, 0.75, 3)
            runs.append(list(r) + [y, k, ctx.dropout_backward(x, k, 0.75)])
        for other in runs[1:]:
            for a, b in zip(runs[0], other):
                assert torch.equal(a, b)
    finally:
        ctx.set_precision("bf16x3")


# ---------------------------------------------------------------------------------------------------- 6. the training demo
def test_lifting_demo_with_dropout_eager_resident_and_graph(tmp_path):
    """--dropout SEED trains with evaluation=False: the device-resident reader and the replayed graph print the eager losses, the graph
    ends with the resident eager run's weights bit for bit, and the weights differ from a run without dropout."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    base = [sys.executable, os.path.join(root, "examples", "train_lifting_demo.py"), "--variant", "proposed", "--augment", "--seed", "3",
            "--iters", "6", "--show-loss-freq", "1"]
    outs, snaps = [], []
    for i, flags in enumerate((["--dropout", "5"], ["--dropout", "5", "--device-resident"], ["--dropout", "5", "--device-resident", "--graph"],
                               ["--device-resident"])):
        snap = tmp_path / ("snap%d" % i)
        r = subprocess.run(base + flags + ["--snapshot-dir", str(snap)], cwd=str(tmp_path), capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
        outs.append([ln for ln in r.stdout.splitlines() if ln.startswith("Iteration")])
        snaps.append((snap / "model-6.pickle").read_bytes())
        print(flags, outs[-1])
    assert len(outs[0]) == 6 and outs[0] == outs[1] == outs[2]
    assert snaps[1] == snaps[2]
    assert snaps[1] != snaps[3]

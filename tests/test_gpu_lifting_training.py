"""GPU training path of the lifting stage (csrc/train_lift.cu, autograd.fully_connected / rotate_canonical / bone_rel_trafo_inv /
mse_loss, PosePriorNetwork.inference(train=True)) against the fp64 lifting oracle (tests/lift_train_oracle.py): the FC layers on
the 1x1 tensor-core path, the new kernels, whole-network gradients of all five variants, training runs, CUDA-graph replay,
snapshots and the readers' 'local' target.

The module runs on a context of its own (installed as the default for its duration), so the weights it loads and trains do not
reach other test modules.  Normwise errors: max|g - ref| / max|ref|."""
import gc
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import lift_train_oracle as L

HERE = os.path.dirname(os.path.abspath(__file__))
pytestmark = pytest.mark.gpu
f32 = np.float32
VARIANTS = ["direct", "bottleneck", "local", "local_w_xyz_loss", "proposed"]
FC_SHAPES = [(2050, 512, True), (512, 512, True), (512, 30, False), (30, 63, False), (512, 63, False), (4098, 256, True),
             (256, 128, True), (128, 3, False)]
FC_TOL = 3 * 5.9e-6            # DESIGN 6.1: the bf16x3 backward's scale-relative error, times three
# A gradient summed over fewer than 32 products (dW at B = 1 and 8, dx of the 128 -> 3 heads) has no long sum to average its
# per-product error over: bf16x3 drops the lo*lo term and the operands' split residuals, up to 2^-15 of |a b| per product
# (DESIGN 4.9; 2.6e-5 measured on an H100 80GB HBM3 at B = 1)
FC_TOL_SHORT = 2.0 ** -15
LIFT_TOL = {"out": 3 * 6.1e-5, "can": 3 * 2.7e-5, "rot": 3 * 6.3e-5}     # DESIGN 6.1, lifting stage, bf16x3, times three
NET_TOL = 7.5e-5               # 3x the largest normwise error over the five variants on an H100 80GB HBM3 (2.4e-5, DESIGN 4.9)


@pytest.fixture(scope="module")
def ctx():
    from hand3d_b200 import runtime
    saved = dict(runtime._default)
    runtime._default.clear()
    c = runtime.default_context()
    c.set_precision("bf16x3")
    yield c
    torch.cuda.synchronize()
    runtime._default.clear()
    runtime._default.update(saved)


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _np(t):
    return t.detach().cpu().numpy()


def _err(g, ref):
    ref = np.asarray(ref, np.float64)
    return float(np.abs(np.asarray(g, np.float64) - ref).max() / max(np.abs(ref).max(), 1e-30))


# ---------------------------------------------------------------------------------------------------- FC through the 1x1 path
@pytest.mark.parametrize("B", [1, 8, 64, 129, 160])
@pytest.mark.parametrize("n_in,n_out,leaky", FC_SHAPES)
def test_fc_gradients_on_the_1x1_path_vs_fp64(ctx, n_in, n_out, leaky, B):
    from hand3d_b200 import autograd as A
    rng = np.random.default_rng(n_in * 7 + n_out + B)
    x = rng.normal(size=(B, n_in)).astype(f32)
    w = (rng.normal(size=(n_in, n_out)) / np.sqrt(n_in)).astype(f32)
    b = (rng.normal(size=n_out) * 0.1).astype(f32)
    dy = rng.normal(size=(B, n_out)).astype(f32)
    xt, wt, bt = _cu(x).requires_grad_(), _cu(w).requires_grad_(), _cu(b).requires_grad_()
    y = A.fully_connected(xt, wt, bt, leaky)
    y.backward(_cu(dy))
    x64, w64, dy64 = x.astype(np.float64), w.astype(np.float64), dy.astype(np.float64)
    z = x64 @ w64 + b
    slope = np.where(_np(y) >= 0, 1.0, 0.01) if leaky else np.ones_like(z)        # the device's leaky decisions
    assert _err(_np(y), z * slope) <= 1e-5
    g = dy64 * slope
    # scale-relative: |d - ref| / (the same sum over absolute values)
    for what, got, ref, scale, K in (("dx", xt.grad, g @ w64.T, np.abs(g) @ np.abs(w64).T, n_out),
                                     ("dw", wt.grad, x64.T @ g, np.abs(x64).T @ np.abs(g), B), ("db", bt.grad, g.sum(0), np.abs(g).sum(0), B)):
        e = np.abs(_np(got) - ref) / np.maximum(scale, 1e-30)
        print("fc %d->%d B=%d %s: %.2e" % (n_in, n_out, B, what, e.max()))
        assert e.max() <= (FC_TOL if K >= 32 else FC_TOL_SHORT), (what, e.max())


# ---------------------------------------------------------------------------------------------------- the new kernels
def _rot_case(seed, B=12, kind="plain"):
    rng = np.random.default_rng(seed)
    can = rng.normal(size=(B, 21, 3)).astype(f32)
    u = rng.normal(size=(B, 3))
    if kind == "small":
        u = u / np.linalg.norm(u, axis=1, keepdims=True) * 1e-5
    if kind == "near_pi":
        u = u / np.linalg.norm(u, axis=1, keepdims=True) * (np.pi - 1e-3)
    hs = np.zeros((B, 2), f32)
    hs[np.arange(B), np.arange(B) % 2] = 1                         # both hands
    return can, u.astype(f32), hs, rng.normal(size=(B, 21, 3)).astype(f32), rng.normal(size=(B, 3, 3)).astype(f32)


@pytest.mark.parametrize("kind", ["plain", "small", "near_pi"])
@pytest.mark.parametrize("which", ["out", "R", "both"])
def test_rotate_canonical_backward_vs_oracle(ctx, which, kind):
    can, u, hs, d_out, d_R = _rot_case(31, kind=kind)
    d_out = d_out if which in ("out", "both") else None
    d_R = d_R if which in ("R", "both") else None
    ref_c, ref_u = L.rotate_canonical_grad(can, u, hs, d_out, d_R)
    args = (_cu(can), _cu(u), _cu(hs), None if d_out is None else _cu(d_out), None if d_R is None else _cu(d_R))
    r1 = ctx.rotate_canonical_backward(*args)
    r2 = ctx.rotate_canonical_backward(*args)
    assert torch.equal(r1[0], r2[0]) and torch.equal(r1[1], r2[1])
    if d_out is None:
        assert not r1[0].any()
    else:
        assert _err(_np(r1[0]), ref_c) <= 1e-6
    assert _err(_np(r1[1]), ref_u) <= 1e-4, _err(_np(r1[1]), ref_u)
    # through autograd: R and out of the forward, either one or both used
    from hand3d_b200 import autograd as A
    ct, ut = _cu(can).requires_grad_(), _cu(u).requires_grad_()
    R, out = A.rotate_canonical(ct, ut, _cu(hs))
    loss = 0
    if d_out is not None:
        loss = loss + (out * _cu(d_out)).sum()
    if d_R is not None:
        loss = loss + (R * _cu(d_R)).sum()
    loss.backward()
    assert torch.equal(ut.grad, r1[1])


def test_bone_rel_trafo_inv_backward_vs_oracle(ctx):
    rng = np.random.default_rng(32)
    rel = np.concatenate([rng.uniform(0.1, 1.0, (9, 21, 1)), rng.uniform(-1.5, 1.5, (9, 21, 2))], 2).astype(f32)
    d = rng.normal(size=(9, 21, 3)).astype(f32)
    g1 = ctx.bone_rel_trafo_inv_backward(_cu(rel), _cu(d))
    g2 = ctx.bone_rel_trafo_inv_backward(_cu(rel), _cu(d))
    assert torch.equal(g1, g2)
    assert _err(_np(g1), L.bone_rel_trafo_inv_grad(rel, d)) <= 1e-5


def test_bone_rel_trafo_vs_oracle_and_reference_graph(ctx):
    G = np.load(os.path.join(HERE, "golden", "golden_reference_graph.npz"))
    r1 = ctx.bone_rel_trafo(_cu(G["coords_xyz"]))
    assert torch.equal(r1, ctx.bone_rel_trafo(_cu(G["coords_xyz"])))
    np.testing.assert_allclose(_np(r1), G["rel_fwd"], rtol=0, atol=2e-5)
    rng = np.random.default_rng(33)
    xyz = rng.normal(size=(17, 21, 3)).astype(f32)
    np.testing.assert_allclose(_np(ctx.bone_rel_trafo(_cu(xyz))), L.bone_rel_trafo(xyz.astype(np.float64)), rtol=0, atol=2e-5)


@pytest.mark.parametrize("shape", [(8, 21, 3), (64, 3, 3), (5000, 7)])
@pytest.mark.parametrize("g", [1.0, -2.5])
def test_mse_vs_fp64_and_reproducible(ctx, shape, g):
    from hand3d_b200 import autograd as A
    rng = np.random.default_rng(34)
    p, t = rng.normal(size=shape).astype(f32), rng.normal(size=shape).astype(f32)
    pt = _cu(p).requires_grad_()
    loss = A.mse_loss(pt, _cu(t))
    loss.backward(torch.tensor(g, device="cuda"))
    assert abs(float(loss) - L.mse(p, t)) <= 1e-6 * L.mse(p, t)
    assert _err(_np(pt.grad), L.mse_grad(p, t, g)) <= 1e-6
    assert torch.equal(ctx.mse_loss(_cu(p), _cu(t)), ctx.mse_loss(_cu(p), _cu(t)))
    assert torch.equal(ctx.mse_loss_backward(_cu(p), _cu(t)), ctx.mse_loss_backward(_cu(p), _cu(t)))


# ---------------------------------------------------------------------------------------------------- whole networks
def _load(ctx, variant, seed=0):
    from hand3d_b200 import weights as Wt
    ctx.load_weights(Wt.xavier_weights(seed, bottleneck=variant == "bottleneck"))


def _batch(seed, B=8):
    """Score maps [B,256,256,21] of Gaussian blobs at random key-points and the reader's targets of random poses."""
    from hand3d_b200 import runtime
    ctx = runtime.default_context()
    rng = np.random.default_rng(seed)
    uv = rng.uniform(20, 236, size=(B, 21, 2)).astype(f32)
    sm = ctx.gaussian_scoremap(_cu(uv), (256, 256), 25.0)
    hs = np.zeros((B, 2), f32)
    hs[np.arange(B), rng.integers(0, 2, B)] = 1
    xyz = (rng.normal(size=(B, 21, 3)) * 0.3).astype(f32)
    t = {"keypoint_xyz21_normed": _cu(xyz), "hand_side": _cu(hs)}
    can, _, rot_inv = ctx.canonical_trafo(t["keypoint_xyz21_normed"], t["hand_side"][:, 1] > 0.5)
    t["keypoint_xyz21_can"], t["rot_mat"] = can, rot_inv
    t["keypoint_xyz21_local"] = ctx.bone_rel_trafo(t["keypoint_xyz21_normed"])
    return sm, t


def _loss(variant, coord3d, R, t):
    """training_lifting.py:62-76."""
    from hand3d_b200 import autograd as A
    from hand3d_b200.utils.relative_trafo import bone_rel_trafo_inv
    if variant in ("direct", "bottleneck"):
        return A.mse_loss(coord3d, t["keypoint_xyz21_normed"])
    if variant == "local":
        return A.mse_loss(coord3d, t["keypoint_xyz21_local"])
    if variant == "local_w_xyz_loss":
        return A.mse_loss(bone_rel_trafo_inv(coord3d), t["keypoint_xyz21_normed"])
    return A.mse_loss(coord3d, t["keypoint_xyz21_can"]) + A.mse_loss(R, t["rot_mat"])


def _scopes(variant):
    return ["PosePrior", "ViewpointNet"] if variant == "proposed" else ["PosePrior"]


class _Decisions:
    """Records every convolution's (and FC layer's) output, whose sign picks the leaky branch: the fp64 reference takes these
    decisions from the device, as tests/test_gpu_training.py does."""

    def __init__(self, monkeypatch):
        from hand3d_b200 import autograd as A
        self.out = []
        conv = A.conv2d

        def rec(x, w, b, stride=1, leaky=True, precision="bf16x3"):
            y = conv(x, w, b, stride, leaky, precision)
            self.out.append(y.detach().cpu().double())
            return y

        monkeypatch.setattr(A, "conv2d", rec)


def _ref_conv(x, w, b, stride, leaky, dec):
    k = w.shape[0]
    xn = x.permute(0, 3, 1, 2)
    if stride == 2:      # TF 'SAME' at stride 2 on even sizes pads only after (total k - 2)
        xn = F.pad(xn, (0, k - 2, 0, k - 2))
        y = F.conv2d(xn, w.permute(3, 2, 0, 1), b, stride=2)
    else:
        y = F.conv2d(xn, w.permute(3, 2, 0, 1), b, padding=k // 2)
    y = y.permute(0, 2, 3, 1)
    y_dev = dec.out.pop(0)
    return torch.where(y_dev >= 0, y, 0.01 * y) if leaky else y


def _ref_fc(x, w, b, leaky, dec):
    y = x @ w + b
    y_dev = dec.out.pop(0).reshape(y.shape)
    return torch.where(y_dev >= 0, y, 0.01 * y) if leaky else y


def _ref_branch(pooled, hs, v, scope, layers, fcs, heads):
    """fp64 restatement of one lifting branch over the Parameters v: conv pyramid, flatten + hand_side, leaky FCs, linear heads."""
    x = pooled
    for name, k, stride, _, _, leaky in layers:
        x = _ref_conv(x, v["%s/%s/weights" % (scope, name)], v["%s/%s/biases" % (scope, name)], stride, leaky, _ref_branch.dec)
    x = torch.cat([x.reshape(x.shape[0], -1), hs], 1)
    for name in fcs:
        x = _ref_fc(x, v["%s/%s/weights" % (scope, name)], v["%s/%s/biases" % (scope, name)], True, _ref_branch.dec)
    for ws, bs in heads:
        x = _ref_fc(x, ws(v), bs(v), False, _ref_branch.dec)
    return x


def _ref_inference(variant, pooled, hs, v, dec):
    from hand3d_b200 import arch
    _ref_branch.dec = dec
    pp = [(lambda v, n=n: v["PosePrior/%s/weights" % n], lambda v, n=n: v["PosePrior/%s/biases" % n])
          for n in (["fc_bottleneck"] if variant == "bottleneck" else []) + ["fc_xyz"]]
    c = _ref_branch(pooled, hs, v, "PosePrior", arch.POSEPRIOR[:6], ["fc_rel0", "fc_rel1"], pp).reshape(-1, 21, 3)
    if variant in ("direct", "bottleneck", "local"):
        return c, None
    if variant == "local_w_xyz_loss":
        return L.bone_rel_trafo_inv_torch(c), None
    heads = [(lambda v: torch.cat([v["ViewpointNet/fc_vp_u%s/weights" % a] for a in "xyz"], 1),
              lambda v: torch.cat([v["ViewpointNet/fc_vp_u%s/biases" % a] for a in "xyz"], 0))]
    u = _ref_branch(pooled, hs, v, "ViewpointNet", arch.VIEWPOINT[:6], ["fc_vp0", "fc_vp1"], heads)
    R, _ = L.rotate_canonical_torch(c, u, hs)
    return c, R


@pytest.mark.parametrize("variant", VARIANTS)
def test_whole_network_gradients_vs_fp64(ctx, variant, monkeypatch):
    from hand3d_b200.nets.PosePriorNetwork import PosePriorNetwork
    _load(ctx, variant)
    v = {}
    for s in _scopes(variant):
        v.update(ctx.variables(s))
    assert len(v) == {"bottleneck": 20, "proposed": 40}.get(variant, 18)
    for p in v.values():
        p.grad = None
    sm, t = _batch(41)
    dec = _Decisions(monkeypatch)
    _, coord3d, R = PosePriorNetwork(variant).inference(sm, t["hand_side"], train=True)
    loss = _loss(variant, coord3d, R, t)
    loss.backward()
    loss = float(loss.detach())
    pooled = ctx.avg_pool8(sm).cpu().double()
    rv = {k: torch.nn.Parameter(p.detach().cpu().double()) for k, p in v.items()}
    tc = {k: x.detach().cpu().double() for k, x in t.items()}
    c_ref, R_ref = _ref_inference(variant, pooled, tc["hand_side"], rv, dec)
    assert not dec.out
    if variant in ("direct", "bottleneck"):
        ref = torch.mean((c_ref - tc["keypoint_xyz21_normed"]) ** 2)
    elif variant == "local":
        ref = torch.mean((c_ref - tc["keypoint_xyz21_local"]) ** 2)
    elif variant == "local_w_xyz_loss":
        ref = torch.mean((c_ref - tc["keypoint_xyz21_normed"]) ** 2)
    else:
        ref = torch.mean((c_ref - tc["keypoint_xyz21_can"]) ** 2) + torch.mean((R_ref - tc["rot_mat"]) ** 2)
    ref.backward()
    assert abs(loss - ref.item()) <= 1e-4 * abs(ref.item()), (loss, ref.item())
    worst = 0.0
    for k, p in v.items():
        assert p.grad is not None and p.grad.abs().max().item() > 0, k
        e = _err(_np(p.grad), rv[k].grad.numpy())
        worst = max(worst, e)
        assert e <= NET_TOL, (k, e)
    print("%s: loss %.6e, worst normwise gradient error %.2e" % (variant, loss, worst))


@pytest.mark.parametrize("variant", VARIANTS)
def test_train_forward_agrees_with_inference(ctx, variant):
    from hand3d_b200.nets.PosePriorNetwork import PosePriorNetwork
    _load(ctx, variant, seed=1)
    sm, t = _batch(42)
    net = PosePriorNetwork(variant)
    with torch.no_grad():
        tr = net.inference(sm, t["hand_side"], train=True)
    inf = net.inference(sm, t["hand_side"])
    assert _err(_np(tr[0]), _np(inf[0]).astype(np.float64)) <= LIFT_TOL["out"]
    assert _err(_np(tr[1]), _np(inf[1]).astype(np.float64)) <= LIFT_TOL["can"]
    if variant == "proposed":
        assert _err(_np(tr[2]), _np(inf[2]).astype(np.float64)) <= LIFT_TOL["rot"]


def test_colorhandpose3d_train_entries(ctx):
    from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork
    from hand3d_b200.nets.PosePriorNetwork import PosePriorNetwork
    _load(ctx, "proposed", seed=2)
    sm, t = _batch(43)
    pooled = ctx.avg_pool8(sm)
    net = ColorHandPose3DNetwork()
    with torch.no_grad():
        out, can, R = PosePriorNetwork("proposed").inference(sm, t["hand_side"], train=True)
        assert torch.equal(net._inference_pose3d(pooled, t["hand_side"], train=True), out)
        assert torch.equal(net._inference_pose3d_can(pooled, t["hand_side"], train=True), can)
        assert torch.equal(net._inference_viewpoint(pooled, t["hand_side"], train=True), R)


# ---------------------------------------------------------------------------------------------------- training behaviour
def _train(ctx, variant, steps, batch, lr=1e-4):
    from hand3d_b200.nets.PosePriorNetwork import PosePriorNetwork
    from hand3d_b200.optim import Adam
    _load(ctx, variant)
    params = [p for s in _scopes(variant) for p in ctx.variables(s).values()]
    opt = Adam(params, lr=lr)
    net = PosePriorNetwork(variant)
    sm, t = batch
    losses = []
    for _ in range(steps):
        opt.zero_grad()
        _, coord3d, R = net.inference(sm, t["hand_side"], train=True)
        loss = _loss(variant, coord3d, R, t)
        loss.backward()
        opt.step()
        losses.append(loss.detach().clone())
    return [float(x) for x in losses], [p.detach().clone() for p in params]


@pytest.mark.parametrize("variant", VARIANTS)
def test_training_lowers_the_loss_and_is_reproducible(ctx, variant):
    batch = _batch(44)
    l1, w1 = _train(ctx, variant, 30, batch)
    l2, w2 = _train(ctx, variant, 30, batch)
    print("%s losses: first %.5e last %.5e" % (variant, l1[0], l1[-1]))
    assert l1[-1] < l1[0]
    assert l1 == l2
    assert all(torch.equal(a, b) for a, b in zip(w1, w2))


def test_cuda_graph_replay_equals_eager_steps(ctx):
    from hand3d_b200.nets.PosePriorNetwork import PosePriorNetwork
    from hand3d_b200.optim import Adam
    sm, t = _batch(45)
    net = PosePriorNetwork("proposed")
    k = 3

    def fresh():
        _load(ctx, "proposed")
        params = [p for s in _scopes("proposed") for p in ctx.variables(s).values()]
        for p in params:
            p.grad = None
        return params, Adam(params, lr=1e-4)

    def step(opt):
        opt.zero_grad()
        _, coord3d, R = net.inference(sm, t["hand_side"], train=True)
        loss = _loss("proposed", coord3d, R, t)
        loss.backward()
        opt.step()

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
        step(opt)
    for _ in range(k):
        g.replay()
    torch.cuda.synchronize()
    for a, b in zip(params, eager):
        assert torch.equal(a.detach(), b)
    del g


def test_train_rejects_fp16_precisions_and_dropout(ctx):
    from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork
    from hand3d_b200.nets.PosePriorNetwork import PosePriorNetwork
    _load(ctx, "proposed")
    sm, t = _batch(46, B=2)
    net = PosePriorNetwork("proposed")
    for prec in ("fp16", "fp16x3", "fp16_f8c", "fp32_ffma"):
        ctx.set_precision(prec)
        try:
            with pytest.raises(ValueError, match="bf16x3"):
                net.inference(sm, t["hand_side"], train=True)
        finally:
            ctx.set_precision("bf16x3")
    with pytest.raises(NotImplementedError):
        net.inference(sm, t["hand_side"], evaluation=False, train=True)
    with pytest.raises(NotImplementedError):
        ColorHandPose3DNetwork()._inference_pose3d(ctx.avg_pool8(sm), t["hand_side"], evaluation=False, train=True)
    with pytest.raises(ValueError, match="bottleneck"):
        PosePriorNetwork("bottleneck").inference(sm, t["hand_side"], train=True)


# ---------------------------------------------------------------------------------------------------- snapshots, commit, readers
def test_snapshot_loads_through_poseprior_init(ctx, tmp_path):
    from hand3d_b200 import weights as Wt
    from hand3d_b200.nets.PosePriorNetwork import PosePriorNetwork
    batch = _batch(47)
    _, _ = _train(ctx, "local_w_xyz_loss", 3, batch)
    path = Wt.save_weight_file(str(tmp_path / "lifting.pickle"), ctx.variables("PosePrior"))
    net = PosePriorNetwork("local")
    with torch.no_grad():
        want = net.inference(batch[0], batch[1]["hand_side"], train=True)
    _load(ctx, "local")                   # back to the initial weights, then the snapshot
    net.init(weight_files=[path])
    got = net.inference(batch[0], batch[1]["hand_side"])
    assert _err(_np(got[1]), _np(want[1]).astype(np.float64)) <= LIFT_TOL["can"]
    assert _err(_np(got[0]), _np(want[0]).astype(np.float64)) <= LIFT_TOL["out"]


def test_commit_variables_updates_inference_including_the_heads(ctx):
    batch = _batch(48)
    sm, t = batch
    pooled = ctx.avg_pool8(sm)
    _train(ctx, "proposed", 3, batch, lr=1e-3)
    from hand3d_b200.nets.PosePriorNetwork import PosePriorNetwork
    with torch.no_grad():
        trained = PosePriorNetwork("proposed").inference(sm, t["hand_side"], train=True)
    stale = ctx.lifting(pooled, t["hand_side"], "proposed")
    assert _err(_np(stale[2]), _np(trained[2]).astype(np.float64)) > 10 * LIFT_TOL["rot"]
    ctx.commit_variables("PosePrior")
    ctx.commit_variables("ViewpointNet")
    fresh = ctx.lifting(pooled, t["hand_side"], "proposed")
    assert _err(_np(fresh[0]), _np(trained[0]).astype(np.float64)) <= LIFT_TOL["out"]
    assert _err(_np(fresh[1]), _np(trained[1]).astype(np.float64)) <= LIFT_TOL["can"]
    assert _err(_np(fresh[2]), _np(trained[2]).astype(np.float64)) <= LIFT_TOL["rot"]


def _write(tmp_path, name, recs):
    p = tmp_path / name
    p.write_bytes(b"".join(recs))
    return str(p)


def test_readers_keypoint_xyz21_local_matches_the_reader_oracle(ctx, tmp_path):
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import synth_records as SR
    from oracle import reader_oracle as R
    from hand3d_b200.data.BinaryDbReader import BinaryDbReader, BinaryDbReaderSTB
    recs = SR.rhd_records(4)
    kw = dict(hand_crop=True, use_wrist_coord=False)
    d = BinaryDbReader(mode="evaluation", shuffle=False, batch_size=4, path_to_db=_write(tmp_path, "rhd.bin", recs), **kw).get()
    for i in range(4):
        np.testing.assert_allclose(_np(d["keypoint_xyz21_local"])[i], R.rhd_items(recs[i], **kw)["keypoint_xyz21_local"], atol=2e-5)
    recs = SR.stb_records(2)
    d = BinaryDbReaderSTB(mode="evaluation", shuffle=False, batch_size=2, path_to_db=_write(tmp_path, "stb.bin", recs)).get()
    for i in range(2):
        np.testing.assert_allclose(_np(d["keypoint_xyz21_local"])[i], R.stb_items(recs[i])["keypoint_xyz21_local"], atol=2e-5)

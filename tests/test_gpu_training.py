"""GPU training path of HandSegNet and PoseNet2D (csrc/train.cu, autograd.py, optim.py, train=True graphs) against the fp64 training
oracle (tests/train_oracle.py): the resize gradient, both losses, TF's Adam bit for bit, whole-network gradients, training runs,
CUDA-graph replay and snapshots.

Errors are normwise: max|g - ref| / max|ref|."""
import copy
import gc

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import train_oracle as O

pytestmark = pytest.mark.gpu
f32 = np.float32

RATIOS = [((32, 32), (256, 256)), ((40, 40), (320, 320)), ((30, 30), (97, 97)), ((17, 17), (5, 5)), ((30, 17), (97, 5)),
          ((24, 20), (24, 20))]
# Whole-network gradients (bf16x3): 3x the normwise errors measured on an H100 80GB HBM3 at 400 W (5.8e-5, 3.9e-5; DESIGN.md 4.8),
# within the 1e-3 cap
NET_TOL = {"PoseNet2D": 1.8e-4, "HandSegNet": 1.2e-4}


@pytest.fixture(scope="module")
def ctx():
    from hand3d_b200 import runtime
    c = runtime.default_context()
    c.set_precision("bf16x3")
    return c


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _err(g, ref):
    return float(np.abs(np.asarray(g, np.float64) - ref).max() / max(np.abs(ref).max(), 1e-30))


# ---------------------------------------------------------------------------------------------------- resize backward
@pytest.mark.parametrize("C", [1, 2, 21, 64])
@pytest.mark.parametrize("B", [1, 3, 8])
@pytest.mark.parametrize("src,dst", RATIOS)
def test_resize_backward_vs_oracle(ctx, src, dst, B, C):
    rng = np.random.default_rng(B * 100 + C)
    dy = rng.normal(size=(B, *dst, C)).astype(f32)
    dx = ctx.resize_bilinear_backward(_cu(dy), *src).cpu().numpy()
    e = _err(dx, O.resize_bilinear_grad(dy, *src))
    assert e <= 1e-6, e


def test_resize_backward_exact_at_ratio_8_and_reproducible(ctx):
    rng = np.random.default_rng(7)
    dy = rng.integers(-8, 9, size=(3, 256, 256, 21)).astype(f32)      # every product with a weight k/8 and every sum is exact
    g = _cu(dy)
    a = ctx.resize_bilinear_backward(g, 32, 32)
    b = ctx.resize_bilinear_backward(g, 32, 32)
    assert np.array_equal(a.cpu().numpy(), O.resize_bilinear_grad(dy, 32, 32).astype(f32))
    assert torch.equal(a, b)
    dy2 = rng.normal(size=(2, 97, 5, 2)).astype(f32)
    r = [ctx.resize_bilinear_backward(_cu(dy2), 30, 17) for _ in range(2)]
    assert torch.equal(r[0], r[1])


def test_resize_backward_rejects_bad_shapes(ctx):
    from hand3d_b200 import _lib
    import ctypes as C
    x = torch.zeros(8, device="cuda")
    assert ctx.lib.h3d_resize_bilinear_tf1_backward(ctx.h, C.c_void_p(x.data_ptr()), C.c_void_p(x.data_ptr()), 1, 0, 2, 1, 2, 2,
                                                     None) == _lib.EINVAL
    assert b"bad shape" in ctx.lib.h3d_last_error()


# ---------------------------------------------------------------------------------------------------- losses
def _scoremap_case(seed, B=3, H=32, W=24):
    rng = np.random.default_rng(seed)
    P = rng.normal(size=(B, H, W, 21)).astype(f32)
    T = rng.normal(size=(B, H, W, 21)).astype(f32)
    vis = (rng.uniform(size=(B, 21)) > 0.3).astype(f32)
    return P, T, vis


@pytest.mark.parametrize("case", ["plain", "vis_row_zero", "vis_all_zero", "rms_zero", "train_shape"])
@pytest.mark.parametrize("g", [1.0, -3.5])
def test_scoremap_loss_vs_fp64(ctx, case, g):
    """train_shape: plain at training_posenet.py's B = 8, 256 x 256, where the reduction runs 33 chunks of 1986 pixels per image."""
    from hand3d_b200 import autograd as A
    P, T, vis = _scoremap_case(11, **(dict(B=8, H=256, W=256) if case == "train_shape" else {}))
    if case == "vis_row_zero":
        vis[1] = 0
    if case == "vis_all_zero":
        vis[:] = 0
    if case == "rms_zero":
        T[0, :, :, 3] = P[0, :, :, 3]
    ref_L, _ = O.scoremap_loss(P, T, vis)
    ref_g = O.scoremap_loss_grad(P, T, vis, g)
    Pt = _cu(P).requires_grad_()
    L = A.scoremap_loss(Pt, _cu(T), _cu(vis))
    L.backward(torch.tensor(g, device="cuda"))
    gpu_L, gpu_g = float(L.detach()), Pt.grad.cpu().numpy()
    if case == "vis_all_zero":
        assert gpu_L == 0.0 and not gpu_g.any()
        return
    print("score-map loss %s, g %g: value %.2e relative, gradient %.2e normwise" % (case, g, abs(gpu_L - ref_L) / abs(ref_L),
                                                                                   _err(gpu_g, ref_g)))
    assert abs(gpu_L - ref_L) <= 1e-5 * abs(ref_L)
    assert np.isfinite(gpu_g).all()
    assert _err(gpu_g, ref_g) <= 1e-5
    if case == "vis_row_zero":
        assert not gpu_g[1].any()
    if case == "rms_zero":
        assert not gpu_g[0, :, :, 3].any()


@pytest.mark.parametrize("labels", ["one_hot", "soft", "unnormalised", "one_hot_train_shape"])
@pytest.mark.parametrize("g", [1.0, 0.25])
def test_softmax_xent_vs_fp64(ctx, labels, g):
    """one_hot_train_shape: one_hot at training_handsegnet.py's B = 8, 256 x 256 (524 288 rows, 256 blocks of 2048)."""
    from hand3d_b200 import autograd as A
    rng = np.random.default_rng(12)
    shape = (8, 256, 256) if labels.endswith("_train_shape") else (3, 40, 24)
    labels = labels.replace("_train_shape", "")
    x = rng.normal(scale=4.0, size=(*shape, 2)).astype(f32)
    if labels == "one_hot":
        hand = rng.uniform(size=shape) > 0.7
        lab = np.stack([~hand, hand], -1).astype(f32)
    else:
        lab = rng.uniform(size=(*shape, 2)).astype(f32)
        if labels == "soft":
            lab = (lab / lab.sum(-1, keepdims=True)).astype(f32)
    xt = _cu(x).requires_grad_()
    L = A.softmax_xent_loss(xt, _cu(lab))
    L.backward(torch.tensor(g, device="cuda"))
    ref_L = O.softmax_xent(x, lab)
    e_L, e_g = abs(float(L.detach()) - ref_L) / abs(ref_L), _err(xt.grad.cpu().numpy(), O.softmax_xent_grad(x, lab, g))
    print("cross-entropy %s %s, g %g: value %.2e relative, gradient %.2e normwise" % (labels, shape, g, e_L, e_g))
    assert e_L <= 1e-5
    assert e_g <= 1e-5


def test_losses_reproducible(ctx):
    P, T, vis = _scoremap_case(13, B=8, H=256, W=256)
    r = [ctx.scoremap_loss(_cu(P), _cu(T), _cu(vis)) for _ in range(2)]
    assert torch.equal(r[0][0], r[1][0]) and torch.equal(r[0][1], r[1][1])
    x = _cu(np.random.default_rng(1).normal(size=(8, 256, 256, 2)).astype(f32))
    lab = torch.stack([x[..., 0] > 0, x[..., 0] <= 0], -1).float()
    assert torch.equal(ctx.softmax_xent(x, lab), ctx.softmax_xent(x, lab))


# ---------------------------------------------------------------------------------------------------- Adam
SIZES = [1, 3, 1025, 10 ** 6]


def _adam_problem(seed=14):
    rng = np.random.default_rng(seed)
    return [rng.normal(size=n).astype(f32) for n in SIZES]


def test_adam_bit_identical_to_tf_restatement_100_steps(ctx):
    from hand3d_b200.optim import Adam
    rng = np.random.default_rng(15)
    init = _adam_problem()
    params = [torch.nn.Parameter(_cu(p.copy())) for p in init]
    opt = Adam(params, lr=1e-3)
    ref = [(p.copy(), np.zeros_like(p), np.zeros_like(p)) for p in init]
    b1p, b2p = np.float32(0.9), np.float32(0.999)
    lr = 1e-3
    for t in range(100):
        if t == 50:
            lr = 3e-4
            opt.set_lr(lr)
        scale = 1e-6 if t % 7 == 3 else 1.0                            # include small-gradient steps (epsilon-hat matters there)
        grads = [(rng.normal(size=p.shape) * scale).astype(f32) for p in init]
        for p, g in zip(params, grads):
            p.grad = _cu(g) if p.grad is None else p.grad.copy_(_cu(g))
        opt.step()
        ref = [O.adam_tf_f32(p, g, m, v, lr, b1p, b2p) for (p, m, v), g in zip(ref, grads)]
        b1p, b2p = O.beta_powers_after(t + 1)
    for p, (rp, rm, rv) in zip(params, ref):
        st = opt.state[p]
        assert np.array_equal(p.detach().cpu().numpy(), rp)
        assert np.array_equal(st["m"].cpu().numpy(), rm) and np.array_equal(st["v"].cpu().numpy(), rv)
    assert opt.beta_powers() == (float(b1p), float(b2p))


def test_adam_state_dict_round_trip(ctx):
    from hand3d_b200.optim import Adam
    rng = np.random.default_rng(16)
    init = _adam_problem(17)

    def run(params, opt, steps, seed):
        r = np.random.default_rng(seed)
        for _ in range(steps):
            for p in params:
                p.grad = _cu(r.normal(size=p.shape).astype(f32))
            opt.step()

    pa = [torch.nn.Parameter(_cu(p.copy())) for p in init]
    oa = Adam(pa, lr=2e-3)
    run(pa, oa, 5, 1)
    sd = copy.deepcopy(oa.state_dict())
    snap = [p.detach().clone() for p in pa]
    run(pa, oa, 4, 2)
    pb = [torch.nn.Parameter(s.clone()) for s in snap]
    ob = Adam(pb, lr=5.0)
    ob.load_state_dict(sd)
    assert ob.param_groups[0]["lr"] == 2e-3
    run(pb, ob, 4, 2)
    for a, b in zip(pa, pb):
        assert torch.equal(a, b)
    assert oa.beta_powers() == ob.beta_powers()
    del rng


def test_adam_rejects_bad_parameters(ctx):
    from hand3d_b200.optim import Adam
    with pytest.raises(TypeError):
        Adam([torch.nn.Parameter(torch.zeros(4))], lr=1e-3)
    with pytest.raises(TypeError):
        Adam([torch.nn.Parameter(torch.zeros(4, dtype=torch.float64, device="cuda"))], lr=1e-3)


# ---------------------------------------------------------------------------------------------------- networks
@pytest.fixture(scope="module")
def net(ctx):
    from hand3d_b200 import weights as Wt
    from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork
    n = ColorHandPose3DNetwork()
    n.init(weights=Wt.synthetic_weights(0))
    return n


class _Decisions:
    """Records the discrete decisions the device took in a train=True graph: every convolution's output (the sign picks the leaky
    branch) and every max-pool input (the window arg-max).  A pre-activation within rounding of 0, or two window entries within
    rounding of each other, is decided by the last bits, and one such element taken differently by the fp64 reference changes a
    whole gradient by O(1 / sqrt(fan-in)).  The reference therefore takes these decisions from the device, as the convolution
    backward tests do with `pre = y`."""

    def __init__(self, monkeypatch):
        from hand3d_b200 import autograd as A
        self.conv_out, self.pool_in = [], []
        conv, pool = A.conv2d, A.max_pool

        def rec_conv(x, w, b, stride=1, leaky=True, precision="bf16x3"):
            y = conv(x, w, b, stride, leaky, precision)
            self.conv_out.append(y.detach().cpu().double())
            return y

        def rec_pool(x):
            self.pool_in.append(x.detach().cpu().double())
            return pool(x)

        monkeypatch.setattr(A, "conv2d", rec_conv)
        monkeypatch.setattr(A, "max_pool", rec_pool)


def _pool_as(x, x_dev):
    """2x2 / 2 max-pool of x that routes each window to the arg-max (first maximum, row-major) of x_dev's window."""
    B, H, W, C = x.shape

    def win(t):
        return t[:, :H // 2 * 2, :W // 2 * 2].reshape(B, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(B, H // 2, W // 2, 4, C)
    idx = torch.argmax(win(x_dev), dim=3, keepdim=True)
    return torch.gather(win(x), 3, idx).squeeze(3)


def _ref_layers(x, v, scope, layers, pool_after, dec):
    for name, k, stride, _, _, leaky in layers:
        w, b = v["%s/%s/weights" % (scope, name)], v["%s/%s/biases" % (scope, name)]
        x = F.conv2d(x.permute(0, 3, 1, 2), w.permute(3, 2, 0, 1), b, padding=k // 2).permute(0, 2, 3, 1)
        y_dev = dec.conv_out.pop(0)
        if leaky:
            x = torch.where(y_dev >= 0, x, 0.01 * x)
        if name in pool_after:
            x = _pool_as(x, dec.pool_in.pop(0))
    return x


def _ref_pose2d(img, v, dec):
    from hand3d_b200 import arch
    L = {l[0]: l for l in arch.POSENET2D}
    trunk = [l for l in arch.POSENET2D if l[0].startswith(("conv1", "conv2", "conv3", "conv4"))]
    enc = _ref_layers(img, v, "PoseNet2D", trunk, arch.POSENET2D_POOL_AFTER, dec)
    maps = [_ref_layers(enc, v, "PoseNet2D", [L["conv5_1"], L["conv5_2"]], (), dec)]
    for u in (6, 7):
        maps.append(_ref_layers(torch.cat([maps[-1], enc], 3), v, "PoseNet2D", [L["conv%d_%d" % (u, i)] for i in range(1, 8)], (), dec))
    assert not dec.conv_out and not dec.pool_in
    return maps


def _ref_detection(img, v, dec):
    from hand3d_b200 import arch
    s = _ref_layers(img, v, "HandSegNet", arch.HANDSEGNET, arch.HANDSEGNET_POOL_AFTER, dec)
    assert not dec.conv_out and not dec.pool_in
    return O.resize_bilinear_torch(s, img.shape[1], img.shape[2])


def _pose_batch(seed=18, B=2, S=64):
    from hand3d_b200 import weights as Wt
    rng = np.random.default_rng(seed)
    img = Wt.synthetic_images(B, S, S, seed=seed)
    target = rng.uniform(size=(B, S, S, 21)).astype(f32) * 0.2
    vis = (rng.uniform(size=(B, 21)) > 0.2).astype(f32)
    return img, target, vis


def _seg_batch(seed=19, B=2, S=64):
    from hand3d_b200 import weights as Wt
    img = Wt.synthetic_images(B, S, S, seed=seed)
    hand = np.random.default_rng(seed).uniform(size=(B, S, S)) > 0.7
    return img, np.stack([~hand, hand], -1).astype(f32)


def _pose_loss(net, img, target, vis):
    from hand3d_b200 import autograd as A
    maps = net.inference_pose2d(img, train=True)
    up = [A.resize_bilinear(m, target.shape[1], target.shape[2]) for m in maps]
    return sum(A.scoremap_loss(u, target, vis) for u in up), maps


def _seg_loss(net, img, labels):
    from hand3d_b200 import autograd as A
    logits = net.inference_detection(img, train=True)[0]
    return A.softmax_xent_loss(logits, labels), logits


def test_pose2d_gradients_vs_fp64(ctx, net, monkeypatch):
    img, target, vis = _pose_batch()
    v, _ = _fresh(ctx, "PoseNet2D")
    assert len(v) == 62
    dec = _Decisions(monkeypatch)
    loss = _pose_loss(net, _cu(img), _cu(target), _cu(vis))[0]
    loss.backward()
    loss = loss.detach()          # keep no autograd node of the device graph alive (see test_cuda_graph_replay_equals_eager_steps)
    rv = {k: torch.nn.Parameter(p.detach().cpu().double()) for k, p in v.items()}
    t64 = torch.from_numpy(target).double()
    ref_loss = sum(O.scoremap_loss_torch(O.resize_bilinear_torch(m, 64, 64), t64, torch.from_numpy(vis).double())
                   for m in _ref_pose2d(torch.from_numpy(img).double(), rv, dec))
    ref_loss.backward()
    errs = {k: _err(v[k].grad.cpu().numpy(), rv[k].grad.numpy()) for k in v}
    worst = max(errs, key=errs.get)
    print("PoseNet2D loss %.6e (fp64 %.6e), worst gradient error %.3e at %s" % (float(loss), float(ref_loss), errs[worst], worst))
    assert abs(float(loss) - float(ref_loss)) <= 1e-4 * abs(float(ref_loss))
    assert errs[worst] <= NET_TOL["PoseNet2D"], errs


def test_detection_gradients_vs_fp64(ctx, net, monkeypatch):
    img, lab = _seg_batch()
    v, _ = _fresh(ctx, "HandSegNet")
    assert len(v) == 32
    dec = _Decisions(monkeypatch)
    loss = _seg_loss(net, _cu(img), _cu(lab))[0]
    loss.backward()
    loss = loss.detach()
    rv = {k: torch.nn.Parameter(p.detach().cpu().double()) for k, p in v.items()}
    ref_loss = O.softmax_xent_torch(_ref_detection(torch.from_numpy(img).double(), rv, dec), torch.from_numpy(lab).double())
    ref_loss.backward()
    errs = {k: _err(v[k].grad.cpu().numpy(), rv[k].grad.numpy()) for k in v}
    worst = max(errs, key=errs.get)
    print("HandSegNet loss %.6e (fp64 %.6e), worst gradient error %.3e at %s" % (float(loss), float(ref_loss), errs[worst], worst))
    assert abs(float(loss) - float(ref_loss)) <= 1e-4 * abs(float(ref_loss))
    assert errs[worst] <= NET_TOL["HandSegNet"], errs


def test_train_forward_agrees_with_inference(ctx, net):
    img, _, _ = _pose_batch(20)
    _fresh(ctx, "PoseNet2D")
    _fresh(ctx, "HandSegNet")
    with torch.no_grad():
        tr = net.inference_pose2d(_cu(img), train=True)
        ev = net.inference_pose2d(_cu(img), train=False)
        seg_tr = net.inference_detection(_cu(img), train=True)[0]
        seg_ev = net.inference_detection(_cu(img), train=False)[0]
    for a, b in zip(tr, ev):
        assert a.shape == b.shape == (2, 8, 8, 21)
        assert (a - b).abs().max().item() <= 1e-3
    assert seg_tr.shape == seg_ev.shape == (2, 64, 64, 2) and (seg_tr - seg_ev).abs().max().item() <= 1e-3


def test_train_rejects_fp16_precisions(ctx, net):
    img = _cu(_pose_batch(21)[0])
    try:
        for prec in ("fp16x3", "fp16", "fp32_ffma"):
            ctx.set_precision(prec)
            with pytest.raises(ValueError, match="bf16x3"):
                net.inference_pose2d(img, train=True)
            with pytest.raises(ValueError, match="bf16"):
                net.inference_detection(img, train=True)
    finally:
        ctx.set_precision("bf16x3")


def test_variables_need_a_loaded_scope():
    from hand3d_b200 import runtime
    c = runtime.Context()
    with pytest.raises(ValueError, match="not loaded"):
        c.variables("PoseNet2D")
    with pytest.raises(ValueError):
        c.variables("PosePrior")


# ---------------------------------------------------------------------------------------------------- wiring, runs, graphs
def _fresh(ctx, scope, seed=0):
    """Resets scope's variables to synthetic_weights(seed) and returns (variables, Adam)."""
    from hand3d_b200 import weights as Wt
    from hand3d_b200.optim import Adam
    w = Wt.synthetic_weights(seed)
    v = ctx.variables(scope)
    with torch.no_grad():
        for k, p in v.items():
            p.copy_(_cu(w[k]))
            p.grad = None
    return v, Adam(list(v.values()), lr=1e-4)


def test_gpu_gradients_through_f32_adam_restatement_match_optim(ctx, net):
    img, target, vis = (_cu(a) for a in _pose_batch(22))
    v, opt = _fresh(ctx, "PoseNet2D")
    loss, _ = _pose_loss(net, img, target, vis)
    loss.backward()
    before = {k: (p.detach().cpu().numpy(), p.grad.cpu().numpy()) for k, p in v.items()}
    opt.step()
    for k, p in v.items():
        rp, _, _ = O.adam_tf_f32(before[k][0], before[k][1], np.zeros_like(before[k][0]), np.zeros_like(before[k][0]), 1e-4, 0.9, 0.999)
        assert np.array_equal(p.detach().cpu().numpy(), rp), k


def _train(ctx, net, scope, steps, batch):
    v, opt = _fresh(ctx, scope)
    losses = []
    for _ in range(steps):
        opt.zero_grad()
        loss = _pose_loss(net, *batch)[0] if scope == "PoseNet2D" else _seg_loss(net, *batch)[0]
        loss.backward()
        opt.step()
        losses.append(loss.detach().clone())
    return [float(l) for l in losses], {k: p.detach().clone() for k, p in v.items()}


@pytest.mark.parametrize("scope", ["PoseNet2D", "HandSegNet"])
def test_training_lowers_the_loss_and_is_reproducible(ctx, net, scope):
    batch = [_cu(a) for a in (_pose_batch(23) if scope == "PoseNet2D" else _seg_batch(23))]
    l1, w1 = _train(ctx, net, scope, 30, batch)
    l2, w2 = _train(ctx, net, scope, 30, batch)
    print("%s losses: first %.5e last %.5e" % (scope, l1[0], l1[-1]))
    assert l1[-1] < l1[0]
    assert l1 == l2
    assert all(torch.equal(w1[k], w2[k]) for k in w1)


def test_cuda_graph_replay_equals_eager_steps(ctx, net):
    img, target, vis = (_cu(a) for a in _pose_batch(24))
    k = 3

    def step(opt):
        opt.zero_grad()
        loss, _ = _pose_loss(net, img, target, vis)
        loss.backward()
        opt.step()
        return loss

    # eager reference: 2 warm-up steps + k steps
    v, opt = _fresh(ctx, "PoseNet2D")
    for _ in range(2 + k):
        step(opt)
    eager = {n: p.detach().clone() for n, p in v.items()}
    # same 2 warm-up steps (they size the scratch and create the gradients), then one captured step replayed k times.  No autograd
    # graph of an earlier step may be alive at capture: its AccumulateGrad nodes would be reused with the stream they were made on.
    v, opt = _fresh(ctx, "PoseNet2D")
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
    for n, p in v.items():
        assert torch.equal(p.detach(), eager[n]), n
    del g


def test_snapshot_loads_for_inference(ctx, net, tmp_path):
    from hand3d_b200 import weights as Wt
    from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork
    batch = [_cu(a) for a in _pose_batch(25)]
    _, trained = _train(ctx, net, "PoseNet2D", 3, batch)
    path = Wt.save_weight_file(str(tmp_path / "posenet.pickle"), trained)
    with torch.no_grad():
        want = net.inference_pose2d(batch[0], train=True)
    n2 = ColorHandPose3DNetwork()
    n2.init(weight_files=[path])
    got = n2.inference_pose2d(batch[0], train=False)
    for a, b in zip(got, want):
        assert (a - b).abs().max().item() <= 1e-3
    init = Wt.synthetic_weights(0)
    assert not np.array_equal(ctx.weights["PoseNet2D/conv1_1/weights"], init["PoseNet2D/conv1_1/weights"])
    net.init(weights=init)         # leave the module's context on the initial weights


def test_commit_variables_and_reload_keep_one_set_of_parameters(ctx, net):
    from hand3d_b200 import weights as Wt
    batch = [_cu(a) for a in _pose_batch(26)]
    v, opt = _fresh(ctx, "PoseNet2D")
    ids = {k: id(p) for k, p in v.items()}
    for _ in range(3):
        opt.zero_grad()
        _pose_loss(net, *batch)[0].backward()
        opt.step()
    with torch.no_grad():
        trained = net.inference_pose2d(batch[0], train=True)
        stale = net.inference_pose2d(batch[0], train=False)          # the inference weights are still the loaded ones
        assert max((a - b).abs().max().item() for a, b in zip(trained, stale)) > 1e-3
        ctx.commit_variables("PoseNet2D")
        fresh = net.inference_pose2d(batch[0], train=False)
    for a, b in zip(fresh, trained):
        assert (a - b).abs().max().item() <= 1e-3
    assert np.array_equal(ctx.weights["PoseNet2D/conv1_1/weights"], v["PoseNet2D/conv1_1/weights"].detach().cpu().numpy())
    # reloading the scope writes into the same Parameters, which the optimiser still holds
    init = Wt.synthetic_weights(0)
    net.init(weights=init)
    v2 = ctx.variables("PoseNet2D")
    assert {k: id(p) for k, p in v2.items()} == ids
    assert all(any(p is q for q in opt.param_groups[0]["params"]) for p in v2.values())
    assert np.array_equal(v2["PoseNet2D/conv4_2/weights"].detach().cpu().numpy(), init["PoseNet2D/conv4_2/weights"])

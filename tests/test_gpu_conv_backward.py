"""GPU backward of the tensor-core convolution and the max-pool (h3d_conv2d_tc_backward, h3d_maxpool2x2_backward_f32, autograd.py)
against the fp64 gradient oracle, with layout canaries, bitwise-reproducibility checks and a small end-to-end SGD run.

Errors are normwise: max|g - ref| / max|ref|."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import tf1_grads as G

pytestmark = pytest.mark.gpu
f32 = np.float32

TOL = {"bf16x3": {"dx": 5e-5, "dw": 1e-4, "db": 1e-4}, "bf16": {"dx": 5e-2, "dw": 5e-2, "db": 5e-2}}

CASES = [  # B, H, W, Cin, Cout, k, stride: the forward's operator cases (stride 1), its stride-2 cases, and backward-specific shapes
    (1, 16, 8, 64, 64, 1, 1), (1, 16, 8, 64, 64, 3, 1), (2, 32, 32, 128, 128, 3, 1), (3, 40, 40, 64, 256, 3, 1),
    (1, 24, 40, 192, 128, 7, 1), (2, 20, 12, 100, 72, 3, 1), (1, 64, 64, 256, 512, 3, 1), (2, 20, 40, 64, 64, 3, 1),
    (3, 64, 64, 64, 64, 3, 1), (2, 24, 48, 64, 128, 3, 1), (4, 80, 80, 128, 256, 3, 1), (1, 24, 16, 64, 64, 3, 1),
    (2, 48, 32, 128, 128, 3, 1),
    (2, 32, 32, 32, 32, 3, 2), (3, 16, 16, 64, 64, 3, 2), (5, 8, 8, 128, 128, 3, 2), (2, 8, 8, 256, 256, 3, 2),
    (1, 12, 20, 21, 40, 3, 2), (2, 32, 32, 64, 64, 3, 2), (2, 32, 32, 128, 128, 3, 2),
    (2, 16, 24, 128, 512, 1, 1),    # k = 1 (conv5_1 / conv6_1 shape)
    (1, 32, 32, 149, 128, 7, 1),    # PoseNet2D conv6_1 / conv7_1: 7x7, 149 -> 128
    (2, 32, 48, 3, 64, 3, 1),       # first layer: Cin = 3, no dx
    (8, 128, 128, 64, 64, 3, 1),    # long K: 131072 pixels per tap
]


@pytest.fixture(scope="module")
def ctx():
    from hand3d_b200 import runtime
    return runtime.default_context()


def _err(g, ref):
    return float(np.abs(np.asarray(g, np.float64) - ref).max() / max(np.abs(ref).max(), 1e-30))


def _problem(case, seed=21):
    B, H, W, Cin, Cout, k, s = case
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(B, H, W, Cin)).astype(f32)
    w = (rng.normal(size=(k, k, Cin, Cout)) / np.sqrt(k * k * Cin)).astype(f32)
    b = rng.normal(size=Cout).astype(f32) * 0.1
    dy = rng.normal(size=(B, H // s, W // s, Cout)).astype(f32)
    return x, w, b, dy


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("prec", ["bf16x3", "bf16"])
@pytest.mark.parametrize("case", CASES)
def test_conv_backward_vs_oracle(ctx, case, prec):
    B, H, W, Cin, Cout, k, s = case
    x, w, b, dy = _problem(case)
    xg, wg, bg, dyg = _cu(x), _cu(w), _cu(b), _cu(dy)
    y = ctx.conv2d_tc_dev(xg, wg, bg, stride=s, leaky=True, precision=prec)
    need_dx = Cin != 3
    dx, dw, db = ctx.conv2d_tc_backward(xg, y, dyg, wg, stride=s, leaky=True, precision=prec, need_dx=need_dx)
    rdx, rdw, rdb = G.conv_grads(x, w, b, dy, s, leaky=True, pre=y.cpu().numpy())
    errs = {"dw": _err(dw.cpu().numpy(), rdw), "db": _err(db.cpu().numpy(), rdb)}
    if need_dx:
        errs["dx"] = _err(dx.cpu().numpy(), rdx)
    else:
        assert dx is None
    for name, e in errs.items():
        assert e < TOL[prec][name], "%s normwise error %.3e (bound %.1e)" % (name, e, TOL[prec][name])


def test_weight_gradient_canary_one_hot_dy(ctx):
    """dy one-hot at one pixel and channel: dW[kh, kw, :, co0] is the x patch around that pixel, every other dW column is zero."""
    B, H, W, Cin, Cout, k = 2, 16, 24, 128, 128, 3
    rng = np.random.default_rng(1)
    x = rng.integers(-4, 5, size=(B, H, W, Cin)).astype(f32)
    w = np.zeros((k, k, Cin, Cout), f32)
    for (b0, h0, w0, co0) in ((1, 5, 9, 70), (0, 0, 23, 3)):   # interior pixel / second M tile; corner pixel (zero padding)
        dy = np.zeros((B, H, W, Cout), f32)
        dy[b0, h0, w0, co0] = 3.0
        for prec in ("bf16x3", "bf16"):
            _, dw, db = ctx.conv2d_tc_backward(_cu(x), None, _cu(dy), _cu(w), leaky=False, precision=prec, need_dx=False)
            ref = np.zeros((k, k, Cin, Cout), f32)
            for kh in range(k):
                for kw in range(k):
                    hh, ww = h0 + kh - 1, w0 + kw - 1
                    if 0 <= hh < H and 0 <= ww < W:
                        ref[kh, kw, :, co0] = 3.0 * x[b0, hh, ww, :]
            np.testing.assert_array_equal(dw.cpu().numpy(), ref)
            assert db.cpu().numpy()[co0] == 3.0 and np.count_nonzero(db.cpu().numpy()) == 1


@pytest.mark.parametrize("stride", [1, 2])
def test_data_gradient_canary_delta_kernel(ctx, stride):
    """w = an off-centre delta tap times a channel permutation: dx must be dy shifted by the tap and permuted, exactly."""
    B, H, W, C, k = 2, 16, 20, 64, 3
    rng = np.random.default_rng(2)
    perm = rng.permutation(C)
    w = np.zeros((k, k, C, C), f32)
    w[0, 2, np.arange(C), perm] = 1.0            # y[p, perm[ci]] = x[p + (-1, +1), ci]
    dy = rng.integers(-8, 9, size=(B, H // stride, W // stride, C)).astype(f32)
    ref = G.conv2d_backprop_input(dy, w, (B, H, W, C), stride)
    for prec in ("bf16x3", "bf16"):
        dx, _, _ = ctx.conv2d_tc_backward(None, None, _cu(dy), _cu(w), stride=stride, leaky=False, precision=prec,
                                          need_dw=False, need_db=False)
        np.testing.assert_array_equal(dx.cpu().numpy(), ref.astype(f32))


def test_backward_is_bitwise_reproducible(ctx):
    case = (3, 40, 40, 64, 256, 3, 1)
    x, w, b, dy = _problem(case)
    xg, wg, bg, dyg = _cu(x), _cu(w), _cu(b), _cu(dy)
    y = ctx.conv2d_tc_dev(xg, wg, bg, leaky=True)
    a = ctx.conv2d_tc_backward(xg, y, dyg, wg, leaky=True)
    c = ctx.conv2d_tc_backward(xg, y, dyg, wg, leaky=True)
    for u, v in zip(a, c):
        assert torch.equal(u, v)


@pytest.mark.parametrize("stride", [1, 2])
def test_data_gradient_does_not_depend_on_the_batch(ctx, stride):
    case = (3, 32, 48, 64, 128, 3, stride)
    x, w, b, dy = _problem(case)
    xg, wg, bg, dyg = _cu(x), _cu(w), _cu(b), _cu(dy)
    y = ctx.conv2d_tc_dev(xg, wg, bg, stride=stride, leaky=True)
    dx3, _, _ = ctx.conv2d_tc_backward(xg, y, dyg, wg, stride=stride, leaky=True, need_dw=False, need_db=False)
    dx1, _, _ = ctx.conv2d_tc_backward(xg[1:2], y[1:2], dyg[1:2], wg, stride=stride, leaky=True, need_dw=False, need_db=False)
    assert torch.equal(dx1[0], dx3[1])


@pytest.mark.parametrize("prec", ["bf16x3", "fp16x3", "fp16", "bf16"])
@pytest.mark.parametrize("case", [(2, 20, 12, 100, 72, 3, 1), (1, 24, 40, 192, 128, 7, 1), (2, 32, 32, 32, 32, 3, 2), (1, 16, 8, 3, 64, 3, 1)])
def test_device_weight_forward_matches_packed(ctx, case, prec):
    x, w, b, _ = _problem(case)
    s = case[6]
    packed = ctx.pack_conv(w, b, precision=prec)
    y_packed = ctx.conv2d_tc_packed(_cu(x), packed, leaky=True, stride=s)
    y_dev = ctx.conv2d_tc_dev(_cu(x), _cu(w), _cu(b), stride=s, leaky=True, precision=prec)
    assert torch.equal(y_dev, y_packed)


def test_cuda_graph_of_forward_and_backward_replays_bitwise(ctx):
    case = (2, 32, 32, 128, 128, 3, 1)
    x, w, b, dy = _problem(case)
    xg, wg, bg, dyg = _cu(x), _cu(w), _cu(b), _cu(dy)

    def step():
        y = ctx.conv2d_tc_dev(xg, wg, bg, leaky=True)
        dx, dw, db = ctx.conv2d_tc_backward(xg, y, dyg, wg, leaky=True)
        p = ctx.max_pool(y)
        dp = ctx.max_pool_backward(y, p)
        return y, dx, dw, db, dp

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        eager = step()                         # also grows the operator scratch to its final size
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    graph.replay()
    torch.cuda.synchronize()
    for u, v in zip(eager, captured):
        assert torch.equal(u, v)


@pytest.mark.parametrize("prec", ["fp16x3", "fp16", "fp16_f8c", "fp32_ffma"])
def test_backward_rejects_other_precisions(ctx, prec):
    from hand3d_b200 import _lib
    x, w, b, dy = _problem((1, 16, 8, 64, 64, 3, 1))
    xg, wg, dyg = _cu(x), _cu(w), _cu(dy)
    dx, dw, db = torch.empty_like(xg), torch.empty_like(wg), torch.empty(64, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())   # noqa: E731
    rc = ctx.lib.h3d_conv2d_tc_backward(ctx.h, p(xg), None, p(dyg), p(wg), p(dx), p(dw), p(db), 1, 16, 8, 64, 64, 3, 1, 0,
                                        _lib.PRECISIONS[prec], C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == _lib.EINVAL
    assert "bf16x3 or bf16" in _lib.last_error()


def test_max_pool_backward_vs_oracle(ctx):
    rng = np.random.default_rng(4)
    x = rng.normal(size=(2, 10, 13, 24)).astype(f32)
    x[0, 0:2, 0:2, :] = 1.5                         # ties: first element of the window
    x[1, 4:6, 6:8, 3] = [[0.0, 2.0], [2.0, 2.0]]
    dy = rng.normal(size=(2, 5, 6, 24)).astype(f32)
    dx = ctx.max_pool_backward(_cu(x), _cu(dy)).cpu().numpy()
    np.testing.assert_array_equal(dx, G.max_pool_grad(x, dy).astype(f32))


# ---------------------------------------------------------------------------------------------- end to end through autograd.py
NET = [(3, 21, 64, True), "pool", (7, 64, 64, True), (1, 64, 21, False)]


def _ref_forward(x, params):
    """fp64 CPU torch forward of NET (NHWC / HWIO, TF 'SAME' for odd k at stride 1 is symmetric)."""
    h = x
    it = iter(params)
    for layer in NET:
        if layer == "pool":
            h = F.max_pool2d(h.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
            continue
        k, _, _, leaky = layer
        w, b = next(it), next(it)
        h = F.conv2d(h.permute(0, 3, 1, 2), w.permute(3, 2, 0, 1), b, padding=k // 2).permute(0, 2, 3, 1)
        if leaky:
            h = torch.maximum(h, 0.01 * h)
    return h


def _gpu_forward(x, params):
    from hand3d_b200 import autograd as A
    h = x
    it = iter(params)
    for layer in NET:
        if layer == "pool":
            h = A.max_pool(h)
            continue
        w, b = next(it), next(it)
        h = A.conv2d(h, w, b, leaky=layer[3])
    return h


def test_sgd_through_autograd_matches_fp64(ctx):
    rng = np.random.default_rng(6)
    init = []
    for layer in NET:
        if layer != "pool":
            k, cin, cout, _ = layer
            init += [(rng.normal(size=(k, k, cin, cout)) / np.sqrt(k * k * cin)).astype(f32), (0.1 * rng.normal(size=cout)).astype(f32)]
    x = rng.normal(size=(2, 32, 32, 21)).astype(f32)
    target = rng.normal(size=(2, 16, 16, 21)).astype(f32)

    def run(params, xx, tt, fwd):
        opt = torch.optim.SGD(params, lr=0.05)
        losses = []
        for _ in range(10):
            opt.zero_grad()
            loss = 0.5 * ((fwd(xx, params) - tt) ** 2).mean()
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
        return losses

    gp = [torch.nn.Parameter(_cu(p)) for p in init]
    gpu_losses = run(gp, _cu(x), _cu(target), _gpu_forward)
    rp = [torch.nn.Parameter(torch.from_numpy(p).double()) for p in init]
    ref_losses = run(rp, torch.from_numpy(x).double(), torch.from_numpy(target).double(), _ref_forward)
    assert gpu_losses[-1] < gpu_losses[0]
    np.testing.assert_allclose(gpu_losses, ref_losses, rtol=1e-4)
    for g, r in zip(gp, rp):
        e = _err(g.detach().cpu().numpy(), r.detach().numpy())
        assert e < 1e-4, "final weights differ from the fp64 run by %.3e (normwise)" % e

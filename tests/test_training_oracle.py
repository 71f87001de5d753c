"""CPU pins of the training oracle (tests/train_oracle.py) and of the host-side training helpers: the resize gradient against the
forward (adjoint identity, torch.autograd), both losses against fp64 torch.autograd and central finite differences, TF's Adam in
float32 and fp64 against each other and against torch.optim.Adam, LearningRateScheduler against the reference, and the snapshot
pickle layout."""
import os
import pickle

import numpy as np
import pytest
import torch

import train_oracle as O
from oracle import tf1_ops

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_reference_lr.npz")
RATIOS = [((32, 32), (256, 256)), ((40, 40), (320, 320)), ((30, 17), (97, 5)), ((17, 30), (5, 97)), ((12, 9), (12, 9)), ((8, 6), (8, 13))]


@pytest.mark.parametrize("src,dst", RATIOS)
def test_resize_grad_is_the_adjoint_of_tf1_ops(src, dst):
    rng = np.random.default_rng(1)
    x = rng.normal(size=(2, *src, 3))
    g = rng.normal(size=(2, *dst, 3))
    Rx = tf1_ops.resize_bilinear_tf1(x, *dst)                    # fp64 input: fp64 index arithmetic
    lhs = float(np.sum(Rx * g))
    rhs = float(np.sum(x * O.resize_bilinear_grad(g, *src, index_dtype=np.float64)))
    assert abs(lhs - rhs) <= 1e-12 * max(1.0, abs(lhs))
    np.testing.assert_allclose(O.resize_bilinear(x, *dst, index_dtype=np.float64), Rx, rtol=0, atol=1e-12)
    # the float32 index arithmetic the device uses agrees with the float32 forward of tf1_ops
    x32 = x.astype(np.float32)
    np.testing.assert_allclose(O.resize_bilinear(x32, *dst), tf1_ops.resize_bilinear_tf1(x32, *dst), rtol=0, atol=1e-5)


@pytest.mark.parametrize("src,dst", RATIOS)
def test_resize_grad_matches_torch_autograd(src, dst):
    rng = np.random.default_rng(2)
    x = torch.tensor(rng.normal(size=(2, *src, 2)), requires_grad=True)
    g = rng.normal(size=(2, *dst, 2))
    y = O.resize_bilinear_torch(x, *dst)
    np.testing.assert_allclose(y.detach().numpy(), O.resize_bilinear(x.detach().numpy(), *dst), atol=1e-12)
    y.backward(torch.from_numpy(g))
    np.testing.assert_allclose(x.grad.numpy(), O.resize_bilinear_grad(g, *src), atol=1e-12)


def _fd(f, x, idx, h=1e-6):
    xp, xm = x.copy(), x.copy()
    xp[idx] += h
    xm[idx] -= h
    return (f(xp) - f(xm)) / (2 * h)


def _scoremap_case(seed=3, B=3, H=6, W=5):
    rng = np.random.default_rng(seed)
    P, T = rng.normal(size=(B, H, W, 21)), rng.normal(size=(B, H, W, 21))
    vis = (rng.uniform(size=(B, 21)) > 0.3).astype(np.float64)
    vis[1] = 0                                                      # a row of invisible key-points
    return P, T, vis


def test_scoremap_loss_matches_torch_and_finite_differences():
    P, T, vis = _scoremap_case()
    L, _ = O.scoremap_loss(P, T, vis)
    Pt = torch.tensor(P, requires_grad=True)
    Lt = O.scoremap_loss_torch(Pt, torch.tensor(T), torch.tensor(vis))
    Lt.backward(torch.tensor(2.5, dtype=torch.float64))
    assert abs(L - float(Lt)) <= 1e-14 * abs(L)
    grad = O.scoremap_loss_grad(P, T, vis, g=2.5)
    np.testing.assert_allclose(grad, Pt.grad.numpy(), rtol=1e-12, atol=1e-16)
    assert not grad[1].any()
    for idx in [(0, 0, 0, 0), (2, 5, 4, 20), (0, 3, 2, 7), (1, 1, 1, 1)]:
        fd = 2.5 * _fd(lambda p: O.scoremap_loss(p, T, vis)[0], P, idx)
        assert abs(fd - grad[idx]) <= 1e-7 * max(1e-3, abs(grad[idx])), (idx, fd, grad[idx])


def test_scoremap_loss_zero_rms_and_zero_vis():
    P, T, vis = _scoremap_case()
    T[0, :, :, 4] = P[0, :, :, 4]                                   # rms 0: TF would give NaN, the library 0
    grad = O.scoremap_loss_grad(P, T, vis)
    assert np.isfinite(grad).all() and not grad[0, :, :, 4].any()
    L, _ = O.scoremap_loss(P, T, np.zeros_like(vis))
    assert L == 0.0 and not O.scoremap_loss_grad(P, T, np.zeros_like(vis)).any()


def test_softmax_xent_matches_torch_and_finite_differences():
    rng = np.random.default_rng(4)
    x = rng.normal(scale=3.0, size=(2, 5, 4, 2))
    lab = rng.uniform(size=(2, 5, 4, 2))                             # soft labels, not one-hot
    lab /= lab.sum(-1, keepdims=True)                                # (TF's backprop is the gradient where each row sums to 1)
    lab[0, 0, 0] = (1.0, 0.0)
    xt = torch.tensor(x, requires_grad=True)
    Lt = O.softmax_xent_torch(xt, torch.tensor(lab))
    Lt.backward(torch.tensor(0.75, dtype=torch.float64))
    assert abs(O.softmax_xent(x, lab) - float(Lt)) <= 1e-13 * abs(float(Lt))
    grad = O.softmax_xent_grad(x, lab, g=0.75)
    np.testing.assert_allclose(grad, xt.grad.numpy(), rtol=1e-12, atol=1e-16)
    for idx in [(0, 0, 0, 0), (1, 4, 3, 1), (0, 2, 1, 1)]:
        fd = 0.75 * _fd(lambda a: O.softmax_xent(a, lab), x, idx)
        assert abs(fd - grad[idx]) <= 1e-7 * max(1e-3, abs(grad[idx]))


def test_adam_f32_restatement_tracks_fp64_and_differs_from_torch():
    rng = np.random.default_rng(5)
    n = 4096
    p0 = rng.normal(size=n).astype(np.float32)
    p32, m32, v32 = p0.copy(), np.zeros(n, np.float32), np.zeros(n, np.float32)
    p64, m64, v64 = p0.astype(np.float64), np.zeros(n), np.zeros(n)
    grads = [rng.normal(size=n).astype(np.float32) for _ in range(20)]
    b1p, b2p = np.float32(0.9), np.float32(0.999)
    for t, g in enumerate(grads):
        p32, m32, v32 = O.adam_tf_f32(p32, g, m32, v32, 1e-3, b1p, b2p)
        p64, m64, v64 = O.adam_tf_f64(p64, g, m64, v64, 1e-3, float(b1p), float(b2p))
        b1p, b2p = O.beta_powers_after(t + 1)
    assert np.abs(p32 - p64).max() <= 1e-6
    # small gradients: TF's epsilon-hat update and torch.optim.Adam's bias-corrected epsilon give visibly different steps
    g = np.full(n, 1e-8, np.float32)
    p_tf, _, _ = O.adam_tf_f64(p0, g, np.zeros(n), np.zeros(n), 1e-3, 0.9, 0.999)
    pt = torch.nn.Parameter(torch.from_numpy(p0.astype(np.float64)))
    opt = torch.optim.Adam([pt], lr=1e-3, betas=(0.9, 0.999), eps=1e-8)
    pt.grad = torch.from_numpy(g.astype(np.float64))
    opt.step()
    step_tf, step_torch = p0 - p_tf, p0 - pt.detach().numpy()
    # TF: m = 0.1 g, sqrt(v) = sqrt(0.001) g, alpha = lr sqrt(0.001) / 0.1; torch: m_hat = g, sqrt(v_hat) = g
    gg = float(g[0])
    np.testing.assert_allclose(step_tf, (0.1 * gg) * (1e-3 * np.sqrt(0.001) / 0.1) / (np.sqrt(0.001) * gg + 1e-8), rtol=1e-9)
    np.testing.assert_allclose(step_torch, 1e-3 * gg / (gg + 1e-8), rtol=1e-6)
    assert np.all(step_torch > 10 * step_tf), (step_tf[0], step_torch[0])


def test_beta_powers_accumulate_in_float32():
    b1p, b2p = O.beta_powers_after(3)
    assert b1p == np.float32(np.float32(np.float32(np.float32(0.9) * np.float32(0.9)) * np.float32(0.9)) * np.float32(0.9))
    assert b2p.dtype == np.float32


def test_learning_rate_scheduler_matches_reference():
    from hand3d_b200.utils.general import LearningRateScheduler
    d = np.load(GOLDEN)
    i = 0
    while "s%d_query" % i in d:
        sched = LearningRateScheduler(steps=[int(s) for s in d["s%d_steps" % i]], values=[float(v) for v in d["s%d_values" % i]])
        got = np.array([sched.get_lr(int(t)) for t in d["s%d_query" % i]], np.float32)
        assert np.array_equal(got, d["s%d_lr" % i]), (i, got, d["s%d_lr" % i])
        i += 1
    assert i == 5


def test_learning_rate_scheduler_boundaries():
    from hand3d_b200.utils.general import LearningRateScheduler
    two = LearningRateScheduler(steps=[10], values=[1.0, 2.0])
    assert [two.get_lr(s) for s in (9, 10, 11)] == [1.0, 1.0, 2.0]                   # strict: step > steps[0]
    three = LearningRateScheduler(steps=[10, 20], values=[1.0, 2.0, 3.0])
    assert [three.get_lr(s) for s in (9, 10, 19, 20)] == [1.0, 2.0, 2.0, 3.0]         # step < steps[0] ... step >= steps[-1]
    assert LearningRateScheduler(steps=[], values=[0.5]).get_lr(123456) == np.float32(0.5)
    assert isinstance(three.get_lr(0), np.float32)
    with pytest.raises(AssertionError):
        LearningRateScheduler(steps=[1, 2], values=[1.0, 2.0])


def test_save_weight_file_writes_the_reference_layout(tmp_path):
    from hand3d_b200 import weights as Wt
    w = {k: v for k, v in Wt.synthetic_weights(0).items() if k.startswith("HandSegNet/")}
    t = {k: torch.from_numpy(v.copy()) for k, v in w.items()}
    path = Wt.save_weight_file(str(tmp_path / "snap.pickle"), t)
    raw = open(path, "rb").read()
    assert raw[:2] == b"\x80\x02"                                                     # pickle protocol 2
    back = pickle.loads(raw)
    assert list(back) == list(w) and all(back[k].dtype == np.float32 and np.array_equal(back[k], w[k]) for k in w)
    loaded = Wt.load_weight_files([path], verbose=False)
    Wt.validate(loaded)
    assert len(loaded) == 32

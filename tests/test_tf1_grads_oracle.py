"""The fp64 gradient oracle (oracle/tf1_grads.py) pinned to two independent sources on the CPU: torch.autograd in fp64 on the TF-'SAME'
convolution (explicit asymmetric F.pad for stride 2), and central finite differences of oracle.tf1_ops.conv2d_same."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import tf1_grads as G
from oracle import tf1_ops as T


def _torch_grads(x, w, b, dy, stride, leaky):
    """(dx, dw, db) by torch.autograd in fp64: NHWC / HWIO in, TF 'SAME' padding written out with F.pad."""
    xt = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    wt = torch.tensor(w, dtype=torch.float64, requires_grad=True)
    bt = torch.tensor(b, dtype=torch.float64, requires_grad=True)
    k = w.shape[0]
    pt, pb = T.same_pad(x.shape[1], k, stride)
    pl, pr = T.same_pad(x.shape[2], k, stride)
    y = F.conv2d(F.pad(xt.permute(0, 3, 1, 2), (pl, pr, pt, pb)), wt.permute(3, 2, 0, 1), bt, stride=stride).permute(0, 2, 3, 1)
    if leaky:
        y = torch.maximum(y, 0.01 * y)
    (y * torch.tensor(dy, dtype=torch.float64)).sum().backward()
    return xt.grad.numpy(), wt.grad.numpy(), bt.grad.numpy()


@pytest.mark.parametrize("case", [  # B, H, W, Cin, Cout, k, stride
    (2, 6, 5, 3, 4, 3, 1),
    (1, 7, 6, 2, 3, 5, 1),
    (2, 4, 4, 3, 2, 1, 1),
    (2, 8, 6, 3, 4, 3, 2),      # stride 2 on an even size: TF pads 0 before, 1 after
    (1, 8, 8, 2, 3, 5, 2),      # k = 5, stride 2: 1 before, 2 after
    (1, 10, 6, 2, 2, 7, 2),
])
@pytest.mark.parametrize("leaky", [False, True])
def test_conv_grads_match_torch_autograd(case, leaky):
    B, H, W, Cin, Cout, k, s = case
    rng = np.random.default_rng(3)
    x = rng.normal(size=(B, H, W, Cin))
    w = rng.normal(size=(k, k, Cin, Cout))
    b = rng.normal(size=Cout)
    dy = rng.normal(size=(B, -(-H // s), -(-W // s), Cout))
    got = G.conv_grads(x, w, b, dy, s, leaky)
    ref = _torch_grads(x, w, b, dy, s, leaky)
    for g, r, name in zip(got, ref, ("dx", "dw", "db")):
        np.testing.assert_allclose(g, r, rtol=1e-12, atol=1e-12, err_msg=name)


@pytest.mark.parametrize("case", [(1, 4, 5, 2, 3, 3, 1), (1, 6, 4, 2, 2, 3, 2), (1, 6, 6, 1, 2, 5, 2)])
def test_conv_grads_match_finite_differences(case):
    """The convolution is linear in x and in w, so central differences of conv2d_same are exact up to rounding."""
    B, H, W, Cin, Cout, k, s = case
    rng = np.random.default_rng(5)
    x = rng.normal(size=(B, H, W, Cin))
    w = rng.normal(size=(k, k, Cin, Cout))
    b = rng.normal(size=Cout)
    dy = rng.normal(size=(B, -(-H // s), -(-W // s), Cout))
    loss = lambda x_, w_, b_: float((T.conv2d_same(x_, w_, b_, s, np.float64) * dy).sum())   # noqa: E731
    dx, dw, db = G.conv_grads(x, w, b, dy, s, leaky=False)
    h = 1e-3
    for arr, grad, which in ((x, dx, 0), (w, dw, 1), (b, db, 2)):
        fd = np.zeros_like(arr)
        for i in np.ndindex(arr.shape):
            args_p, args_m = [x.copy(), w.copy(), b.copy()], [x.copy(), w.copy(), b.copy()]
            args_p[which][i] += h
            args_m[which][i] -= h
            fd[i] = (loss(*args_p) - loss(*args_m)) / (2 * h)
        np.testing.assert_allclose(grad, fd, rtol=1e-8, atol=1e-8)


def test_leaky_relu_grad_routes_like_tf_maximum():
    pre = np.array([-2.0, -0.0, 0.0, 3.0])
    dy = np.array([1.0, 2.0, 3.0, 4.0])
    np.testing.assert_array_equal(G.leaky_relu_grad(pre, dy), [0.01, 2.0, 3.0, 4.0])


def test_max_pool_grad_ties_go_to_first_element():
    x = np.zeros((1, 4, 5, 2))
    x[0, 0:2, 0:2, 0] = 1.0                 # four-way tie: the top-left element takes it
    x[0, 0:2, 2:4, 0] = [[0.0, 2.0], [2.0, 0.0]]   # tie between (0, 1) and (1, 0): (0, 1) comes first in row-major order
    x[0, 2, 2, 1] = 5.0
    x[0, 2:4, 4, :] = 9.0                   # the fifth column is dropped by the VALID pool
    dy = np.arange(1, 1 + 2 * 2 * 2, dtype=np.float64).reshape(1, 2, 2, 2)
    dx = G.max_pool_grad(x, dy)
    assert dx[0, 0, 0, 0] == dy[0, 0, 0, 0] and dx[0, 0:2, 0:2, 0].sum() == dy[0, 0, 0, 0]
    assert dx[0, 0, 3, 0] == dy[0, 0, 1, 0] and dx[0, 1, 2, 0] == 0.0
    assert dx[0, 2, 2, 1] == dy[0, 1, 1, 1]
    assert not dx[0, :, 4, :].any()
    assert dx.sum() == dy.sum()


def test_max_pool_grad_matches_torch_without_ties():
    rng = np.random.default_rng(9)
    x = rng.normal(size=(2, 6, 7, 3))
    dy = rng.normal(size=(2, 3, 3, 3))
    xt = torch.tensor(x, requires_grad=True)
    y = F.max_pool2d(xt.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
    (y * torch.tensor(dy)).sum().backward()
    np.testing.assert_array_equal(G.max_pool_grad(x, dy), xt.grad.numpy())
    np.testing.assert_array_equal(y.detach().numpy(), T.max_pool_2x2(x))

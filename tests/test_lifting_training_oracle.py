"""CPU pins of the lifting-training oracle (tests/lift_train_oracle.py): the hand-written adjoints of Rodrigues + flip + rotate,
of the forward kinematics and of the MSE against fp64 torch.autograd and central finite differences; bone_rel_trafo against the
reference's own graph (golden_reference_graph.npz); and the Xavier initialiser's shapes and ranges."""
import os

import numpy as np
import pytest
import torch

import lift_train_oracle as L

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_reference_graph.npz"))


def _case(seed, B=4, scale=1.0):
    rng = np.random.default_rng(seed)
    can = rng.normal(size=(B, 21, 3))
    u = rng.normal(size=(B, 3)) * scale
    hs = np.zeros((B, 2))
    hs[np.arange(B), np.arange(B) % 2] = 1
    return can, u, hs, rng.normal(size=(B, 21, 3)), rng.normal(size=(B, 3, 3))


def _autograd_rotate(can, u, hs, d_out, d_R):
    c = torch.tensor(can, requires_grad=True)
    v = torch.tensor(u, requires_grad=True)
    R, out = L.rotate_canonical_torch(c, v, torch.tensor(hs))
    loss = 0
    if d_out is not None:
        loss = loss + (out * torch.tensor(d_out)).sum()
    if d_R is not None:
        loss = loss + (R * torch.tensor(d_R)).sum()
    loss.backward()
    return (np.zeros_like(can) if c.grad is None else c.grad.numpy()), v.grad.numpy()


def test_rotate_canonical_forward_matches_the_oracle_and_the_torch_form():
    can, u, hs, _, _ = _case(1)
    R, out = L.rotate_canonical(can, u, hs)
    Rt, outt = L.rotate_canonical_torch(torch.tensor(can), torch.tensor(u), torch.tensor(hs))
    np.testing.assert_allclose(R, Rt.numpy(), atol=1e-14)
    np.testing.assert_allclose(out, outt.numpy(), atol=1e-13)
    np.testing.assert_allclose(out[1] @ np.linalg.inv(R[1]), can[1] * [1, 1, -1], atol=1e-12)     # sample 1 is a right hand
    np.testing.assert_allclose(out[0] @ np.linalg.inv(R[0]), can[0], atol=1e-12)


@pytest.mark.parametrize("which", ["out", "R", "both"])
@pytest.mark.parametrize("scale", [1.0, 1e-5, np.pi / np.sqrt(3) * 0.9999])
def test_rotate_canonical_grad_vs_autograd(which, scale):
    can, u, hs, d_out, d_R = _case(2, scale=scale)
    if scale > 1.5:                                   # |u| near pi
        u = u / np.linalg.norm(u, axis=1, keepdims=True) * (np.pi - 1e-3)
    d_out = d_out if which in ("out", "both") else None
    d_R = d_R if which in ("R", "both") else None
    dc, du = L.rotate_canonical_grad(can, u, hs, d_out, d_R)
    rc, ru = _autograd_rotate(can, u, hs, d_out, d_R)
    np.testing.assert_allclose(dc, rc, atol=1e-12)
    np.testing.assert_allclose(du, ru, rtol=1e-9, atol=1e-9 * np.abs(ru).max())


def test_rotate_canonical_grad_vs_finite_differences():
    can, u, hs, d_out, d_R = _case(3)
    _, du = L.rotate_canonical_grad(can, u, hs, d_out, d_R)
    h = 1e-6
    for b in range(len(u)):
        for i in range(3):
            up, um = u.copy(), u.copy()
            up[b, i] += h
            um[b, i] -= h
            f = [(L.rotate_canonical(can, x, hs)[1] * d_out).sum() + (L.rotate_canonical(can, x, hs)[0] * d_R).sum() for x in (up, um)]
            assert abs((f[0] - f[1]) / (2 * h) - du[b, i]) <= 1e-6 * max(1.0, abs(du[b, i]))


def test_bone_rel_trafo_inv_torch_form_and_grad_vs_autograd():
    rng = np.random.default_rng(4)
    rel = np.concatenate([rng.uniform(0.1, 1.0, (3, 21, 1)), rng.uniform(-1.5, 1.5, (3, 21, 2))], 2)
    d = rng.normal(size=(3, 21, 3))
    r = torch.tensor(rel, requires_grad=True)
    xyz = L.bone_rel_trafo_inv_torch(r)
    np.testing.assert_allclose(xyz.detach().numpy(), L.bone_rel_trafo_inv(rel), atol=1e-12)
    (xyz * torch.tensor(d)).sum().backward()
    np.testing.assert_allclose(L.bone_rel_trafo_inv_grad(rel, d), r.grad.numpy(), atol=1e-11)


def test_bone_rel_trafo_inv_grad_vs_finite_differences():
    rng = np.random.default_rng(5)
    rel = np.concatenate([rng.uniform(0.1, 1.0, (2, 21, 1)), rng.uniform(-1.5, 1.5, (2, 21, 2))], 2)
    d = rng.normal(size=(2, 21, 3))
    g = L.bone_rel_trafo_inv_grad(rel, d)
    h = 1e-6
    for idx in [(0, 0, 0), (0, 4, 1), (1, 1, 2), (1, 17, 0), (0, 9, 2), (1, 13, 1)]:
        p, m = rel.copy(), rel.copy()
        p[idx] += h
        m[idx] -= h
        fd = ((L.bone_rel_trafo_inv(p) - L.bone_rel_trafo_inv(m)) * d).sum() / (2 * h)
        assert abs(fd - g[idx]) <= 1e-6 * max(1.0, abs(g[idx])), idx


def test_bone_rel_trafo_matches_the_reference_graph():
    np.testing.assert_allclose(L.bone_rel_trafo(G["coords_xyz"]), G["rel_fwd"], rtol=0, atol=2e-5)
    np.testing.assert_allclose(L.bone_rel_trafo_inv(L.bone_rel_trafo(G["coords_xyz"].astype(np.float64))), G["coords_xyz"], atol=1e-6)


@pytest.mark.parametrize("g", [1.0, -0.5])
def test_mse_grad_vs_autograd_and_finite_differences(g):
    rng = np.random.default_rng(6)
    p, t = rng.normal(size=(5, 21, 3)), rng.normal(size=(5, 21, 3))
    pt = torch.tensor(p, requires_grad=True)
    loss = torch.mean((pt - torch.tensor(t)) ** 2)
    assert abs(loss.item() - L.mse(p, t)) <= 1e-14
    (loss * g).backward()
    np.testing.assert_allclose(L.mse_grad(p, t, g), pt.grad.numpy(), atol=1e-15)
    h = 1e-6
    q, r = p.copy(), p.copy()
    q[2, 7, 1] += h
    r[2, 7, 1] -= h
    assert abs(g * (L.mse(q, t) - L.mse(r, t)) / (2 * h) - L.mse_grad(p, t, g)[2, 7, 1]) <= 1e-8


def test_xavier_weights_shapes_and_ranges():
    from hand3d_b200 import arch
    from hand3d_b200 import weights as Wt
    w = Wt.xavier_weights(0, bottleneck=True)
    shapes = arch.variable_shapes(True)
    assert sorted(w) == sorted(k for k in shapes if k.split("/")[0] in ("PosePrior", "ViewpointNet"))
    assert len([k for k in w if k.startswith("PosePrior/")]) == 20 and len([k for k in w if k.startswith("ViewpointNet/")]) == 22
    for k, a in w.items():
        assert a.shape == shapes[k] and a.dtype == np.float32
        if k.endswith("/biases"):
            assert (a == np.float32(1e-4)).all()
        else:
            s = shapes[k]
            rf = int(np.prod(s[:-2])) if len(s) > 2 else 1
            lim = np.sqrt(6.0 / (rf * (s[-2] + s[-1])))
            assert np.abs(a).max() <= lim and np.abs(a).max() > 0.9 * lim
            assert abs(a.var() - lim ** 2 / 3) <= 0.2 * lim ** 2 / 3 or a.size < 200
    assert np.array_equal(Wt.xavier_weights(3)["PosePrior/fc_rel0/weights"], Wt.xavier_weights(3)["PosePrior/fc_rel0/weights"])
    assert "PosePrior/fc_bottleneck/weights" not in Wt.xavier_weights(0)

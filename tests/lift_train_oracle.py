"""fp64 oracle of the lifting stage's training pieces (training_lifting.py, nets/PosePriorNetwork.py:59-159,
utils/relative_trafo.py): the Rodrigues rotation + right-hand flip + rotate of the 'proposed' variant, the forward kinematics
bone_rel_trafo_inv and its analysis bone_rel_trafo, and the mean squared error, each with a hand-written adjoint.

Every function has two forms: numpy (the adjoints, written out as csrc/train_lift.cu computes them) and torch (differentiable, for
torch.autograd and for the whole-network reference graphs).  tests/test_lifting_training_oracle.py pins the adjoints to torch fp64
autograd and to central finite differences."""
import numpy as np
import torch

from oracle import hand3d_oracle as _H

CHAINS = [[0], [4, 3, 2, 1], [8, 7, 6, 5], [12, 11, 10, 9], [16, 15, 14, 13], [20, 19, 18, 17]]   # kinematic_chain_list by chain


# ---------------------------------------------------------------------------------------------------- Rodrigues + flip + rotate
def _right(hand_side):
    hs = np.asarray(hand_side)
    return hs[:, 1] > hs[:, 0]            # argmax(hand_side, 1) == 1, ties -> index 0


def rodrigues(u):
    """nets/PosePriorNetwork.py:161-184: u [B,3] -> R [B,3,3]."""
    u = np.asarray(u, np.float64)
    th = np.sqrt((u ** 2).sum(1) + 1e-8)
    n = u / th[:, None]
    st, ct = np.sin(th), np.cos(th)
    E = np.zeros((len(u), 3, 3))
    E[:, 0, 1], E[:, 0, 2], E[:, 1, 0], E[:, 1, 2], E[:, 2, 0], E[:, 2, 1] = -n[:, 2], n[:, 1], n[:, 2], -n[:, 0], -n[:, 1], n[:, 0]
    return ct[:, None, None] * np.eye(3) + (1 - ct)[:, None, None] * n[:, :, None] * n[:, None, :] + st[:, None, None] * E


def rotate_canonical(can, u, hand_side):
    """-> (R [B,3,3], out [B,21,3] = flip(can) R)."""
    R = rodrigues(u)
    c = np.array(can, np.float64)
    c[_right(hand_side), :, 2] *= -1
    return R, c @ R


def rotate_canonical_grad(can, u, hand_side, d_out=None, d_R=None):
    """Adjoint of rotate_canonical: -> (d_can [B,21,3], d_u [B,3]); d_out / d_R None count as zero."""
    u = np.asarray(u, np.float64)
    B = len(u)
    R = rodrigues(u)
    s = np.ones((B, 1, 3))
    s[_right(hand_side), 0, 2] = -1
    c = np.asarray(can, np.float64) * s
    d_out = np.zeros((B, 21, 3)) if d_out is None else np.asarray(d_out, np.float64)
    G = (np.zeros((B, 3, 3)) if d_R is None else np.asarray(d_R, np.float64)) + c.transpose(0, 2, 1) @ d_out
    d_can = (d_out @ R.transpose(0, 2, 1)) * s
    th = np.sqrt((u ** 2).sum(1) + 1e-8)
    n = u / th[:, None]
    st, ct = np.sin(th), np.cos(th)
    d_ct = np.trace(G, axis1=1, axis2=2)
    d_one_ct = np.einsum("bij,bi,bj->b", G, n, n)
    e = np.stack([G[:, 2, 1] - G[:, 1, 2], G[:, 0, 2] - G[:, 2, 0], G[:, 1, 0] - G[:, 0, 1]], 1)
    d_st = (e * n).sum(1)
    d_n = (1 - ct)[:, None] * np.einsum("bij,bj->bi", G + G.transpose(0, 2, 1), n) + st[:, None] * e
    d_nf = (d_n * u).sum(1)
    d_th = (d_one_ct - d_ct) * st + d_st * ct - d_nf / th ** 2
    d_u = d_n / th[:, None] + (d_th / th)[:, None] * u
    return d_can, d_u


def rotate_canonical_torch(can, u, hand_side):
    """Differentiable torch form (any dtype) -> (R, out)."""
    th = torch.sqrt((u ** 2).sum(1) + 1e-8)
    n = u / th[:, None]
    st, ct = torch.sin(th), torch.cos(th)
    z = torch.zeros_like(th)
    E = torch.stack([z, -n[:, 2], n[:, 1], n[:, 2], z, -n[:, 0], -n[:, 1], n[:, 0], z], 1).view(-1, 3, 3)
    I = torch.eye(3, dtype=u.dtype, device=u.device)
    R = ct[:, None, None] * I + (1 - ct)[:, None, None] * n[:, :, None] * n[:, None, :] + st[:, None, None] * E
    right = hand_side[:, 1] > hand_side[:, 0]
    s = torch.ones((len(u), 1, 3), dtype=u.dtype, device=u.device)
    s[right, 0, 2] = -1
    return R, (can * s) @ R


# ---------------------------------------------------------------------------------------------------- forward kinematics
def _rot_xy(a, b):
    """RotX(a) RotY(b) (3x3, the rotation part of the reference's _forward)."""
    ca, sa, cb, sb = np.cos(a), np.sin(a), np.cos(b), np.sin(b)
    return np.array([[cb, 0, sb], [sa * sb, ca, -sa * cb], [-ca * sb, sa, ca * cb]])


def bone_rel_trafo_inv(rel):
    """utils/relative_trafo.py:243-295 (fp64): rel [B,21,3] -> xyz [B,21,3]."""
    return _H.bone_rel_trafo_inv(np.asarray(rel, np.float64))


def bone_rel_trafo_inv_grad(rel, d_xyz):
    """Adjoint of bone_rel_trafo_inv, per chain in reverse: R <- M R, t <- M t - len e_z, x = -R^T t."""
    rel = np.asarray(rel, np.float64).reshape(-1, 21, 3)
    d_xyz = np.asarray(d_xyz, np.float64).reshape(rel.shape)
    d_rel = np.zeros_like(rel)
    for b in range(len(rel)):
        for chain in CHAINS:
            states = []
            R, t = np.eye(3), np.zeros(3)
            for bone in chain:
                states.append((R, t))
                M = _rot_xy(-rel[b, bone, 1], -rel[b, bone, 2])
                R, t = M @ R, M @ t - np.array([0, 0, rel[b, bone, 0]])
            dR, dt = np.zeros((3, 3)), np.zeros(3)
            for i in reversed(range(len(chain))):
                bone = chain[i]
                g = d_xyz[b, bone]
                dR -= np.outer(t, g)
                dt -= R @ g
                Rp, tp = states[i]
                a, c = -rel[b, bone, 1], -rel[b, bone, 2]
                M = _rot_xy(a, c)
                dM = dR @ Rp.T + np.outer(dt, tp)
                ca, sa, cb, sb = np.cos(a), np.sin(a), np.cos(c), np.sin(c)
                dMa = np.array([[0, 0, 0], [ca * sb, -sa, -ca * cb], [sa * sb, ca, -sa * cb]])
                dMb = np.array([[-sb, 0, cb], [sa * cb, 0, sa * sb], [-ca * cb, 0, -ca * sb]])
                d_rel[b, bone] = (-dt[2], -(dM * dMa).sum(), -(dM * dMb).sum())
                dR, dt = M.T @ dR, M.T @ dt
                R, t = Rp, tp
    return d_rel


def bone_rel_trafo_inv_torch(rel):
    """Differentiable torch form: rel [B,21,3] -> xyz [B,21,3]."""
    B = rel.shape[0]
    out = [None] * 21
    for chain in CHAINS:
        R = torch.eye(3, dtype=rel.dtype, device=rel.device).expand(B, 3, 3)
        t = torch.zeros((B, 3), dtype=rel.dtype, device=rel.device)
        for bone in chain:
            a, c = -rel[:, bone, 1], -rel[:, bone, 2]
            ca, sa, cb, sb = torch.cos(a), torch.sin(a), torch.cos(c), torch.sin(c)
            z = torch.zeros_like(a)
            M = torch.stack([cb, z, sb, sa * sb, ca, -sa * cb, -ca * sb, sa, ca * cb], 1).view(B, 3, 3)
            R = M @ R
            t = (M @ t[:, :, None])[:, :, 0] - torch.stack([z, z, rel[:, bone, 0]], 1)
            out[bone] = -(R.transpose(1, 2) @ t[:, :, None])[:, :, 0]
    return torch.stack(out, 1)


def bone_rel_trafo(xyz):
    """utils/relative_trafo.py:184-240 with the reference's atan2, in the dtype of xyz."""
    return _H.bone_rel_trafo(np.asarray(xyz))


# ---------------------------------------------------------------------------------------------------- MSE
def mse(p, t):
    return float(np.mean((np.asarray(p, np.float64) - np.asarray(t, np.float64)) ** 2))


def mse_grad(p, t, g=1.0):
    p, t = np.asarray(p, np.float64), np.asarray(t, np.float64)
    return g / p.size * 2 * (p - t)

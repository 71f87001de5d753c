"""Function-preserving rescaling of the four networks' weights (test infrastructure only).

Leaky ReLU and the 2x2 max-pool are positively homogeneous per channel: act(2^e z) = 2^e act(z).  Scaling the weight column
and the bias of a hidden output channel by 2^e therefore scales that channel's activation by exactly 2^e, and scaling the
matching input rows of every layer that reads the channel by 2^-e restores each product term exactly.  The rescaled
network computes the same function, while the magnitudes its layers see span 2^-E .. 2^E from channel to channel: what
trained weights look like and what He-init weights (hand3d_b200.weights.synthetic_weights) never show.

Where channels meet:
  * PoseNet2D conv4_7 (the encoding) feeds conv5_1, conv6_1 and conv7_1; conv6_1 / conv7_1 read concat([scores, enc]), so
    only their input channels 21..148 are compensated.
  * The FC stacks read the flattened HWC map of the last pyramid layer plus 2 hand_side rows: row p*C + c belongs to channel c;
    the hand_side rows are left alone.
  * Score-producing layers (HandSegNet conv6_2, PoseNet2D conv5_2 / conv6_7 / conv7_7, the final FC layers) keep their scale.
"""
import numpy as np

_HANDSEG = ["conv1_1", "conv1_2", "conv2_1", "conv2_2", "conv3_1", "conv3_2", "conv3_3", "conv3_4", "conv4_1", "conv4_2", "conv4_3",
            "conv4_4", "conv5_1", "conv5_2", "conv6_1", "conv6_2"]
_POSE_TRUNK = ["conv1_1", "conv1_2", "conv2_1", "conv2_2", "conv3_1", "conv3_2", "conv3_3", "conv3_4", "conv4_1", "conv4_2", "conv4_3",
               "conv4_4", "conv4_5", "conv4_6", "conv4_7"]


def _chain(names):
    return [(a, [(b, 0, 0)]) for a, b in zip(names[:-1], names[1:])]


def graph(scope):
    """[(layer, [(consumer, first input channel or row, pixels per channel of an FC flatten or 0)])]; unlisted layers keep their scale"""
    if scope == "HandSegNet":
        return _chain(_HANDSEG)
    if scope == "PoseNet2D":
        g = _chain(_POSE_TRUNK)
        g.append(("conv4_7", [("conv5_1", 0, 0), ("conv6_1", 21, 0), ("conv7_1", 21, 0)]))
        g.append(("conv5_1", [("conv5_2", 0, 0)]))
        for u in (6, 7):
            g += _chain(["conv%d_%d" % (u, i) for i in range(1, 8)])
        return g
    if scope in ("PosePrior", "ViewpointNet"):
        p = "conv_pose_" if scope == "PosePrior" else "conv_vp_"
        convs = ["%s%d_%d" % (p, i, j) for i in range(3) for j in (1, 2)]
        g = _chain(convs)
        if scope == "PosePrior":
            g.append((convs[-1], [("fc_rel0", 0, 16)]))   # 4x4 pixels of the last pyramid layer
            g += [("fc_rel0", [("fc_rel1", 0, 0)]), ("fc_rel1", [("fc_xyz", 0, 0)])]
        else:
            g.append((convs[-1], [("fc_vp0", 0, 16)]))
            g += [("fc_vp0", [("fc_vp1", 0, 0)]), ("fc_vp1", [("fc_vp_ux", 0, 0), ("fc_vp_uy", 0, 0), ("fc_vp_uz", 0, 0)])]
        return g
    raise ValueError(scope)


def rescale(weights, E, seed=0, scopes=("HandSegNet", "PoseNet2D", "PosePrior", "ViewpointNet")):
    """Copy of `weights` with every hidden output channel of `scopes` scaled by 2^e, e uniform in [-E, E] per channel, and its
    consumers compensated by 2^-e.  Exact in any binary floating-point type as long as nothing over- or underflows.
    Returns (weights, {scope/layer: exponents})."""
    rng = np.random.default_rng(seed)
    out = {k: np.array(v, copy=True) for k, v in weights.items()}
    exps = {}
    for scope in scopes:
        for layer, consumers in graph(scope):
            w = out["%s/%s/weights" % (scope, layer)]
            C = w.shape[-1]
            e = rng.integers(-E, E + 1, size=C)
            s = np.ldexp(np.ones(C), e).astype(w.dtype)
            w *= s
            out["%s/%s/biases" % (scope, layer)] *= s
            for cons, off, pix in consumers:
                cw = out["%s/%s/weights" % (scope, cons)]
                if cw.ndim == 4:   # conv HWIO: input channels [off, off + C)
                    cw[:, :, off:off + C, :] /= s[None, None, :, None]
                else:              # FC [in, out]: rows p*C + c of the flattened HWC map
                    pix = max(pix, 1)
                    v = cw[off:off + pix * C].reshape(pix, C, -1)
                    v /= s[None, :, None]
            exps["%s/%s" % (scope, layer)] = e
    return out, exps

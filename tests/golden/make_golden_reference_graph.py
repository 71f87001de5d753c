"""Golden tensors produced by running the reference's own GRAPH-BUILDING code (unmodified, imported from a checkout of lmb-freiburg/hand3d ($H3D_REFERENCE)) over an
eager numpy stand-in for `tensorflow` (oracle/tf1_eager.py).

What this pins and what it does not: the layer lists, variable names and shapes, strides, pool positions, concat order, mask growing
loop, bounding-box / crop arithmetic, Rodrigues formula, right-hand flip, kinematic chain and return-tuple orders are executed from
the REFERENCE source; the heavy ops underneath (conv2d, pools, legacy bilinear resize, soft-max, dilation2d, crop_and_resize) are the
oracle's restatement of the published TF 1.3 kernels (oracle/tf1_ops.py), because TensorFlow itself cannot run here.  So the stored
tensors pin oracle/hand3d_oracle.py's restatement of the GRAPH (and through it the CUDA path) to the reference source; the op
semantics stay pinned by the known-answer tests only.

    python tests/golden/make_golden_reference_graph.py        # H3D_REFERENCE=<checkout of lmb-freiburg/hand3d>; ~1 minute of CPU
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("H3D_REFERENCE", "")   # a checkout of lmb-freiburg/hand3d (needed only to regenerate)
OUT = os.path.join(HERE, "golden_reference_graph.npz")


def setup_imports():
    """`tensorflow` -> the eager stand-in; top-level `nets` / `utils` -> the REFERENCE packages (not this repo's import shims)."""
    sys.path[:] = [p for p in sys.path if os.path.abspath(p or ".") not in (ROOT, HERE)]
    sys.path.insert(0, REF)
    sys.path.append(ROOT)
    import oracle.tf1_eager as tfe
    py = types.ModuleType("tensorflow.python")
    py.pywrap_tensorflow = types.ModuleType("tensorflow.python.pywrap_tensorflow")
    tfe.python = py
    sys.modules["tensorflow"] = tfe
    sys.modules["tensorflow.python"] = py
    sys.modules["tensorflow.python.pywrap_tensorflow"] = py.pywrap_tensorflow
    # the reference's `nets` / `utils` directories have no __init__.py (Python 2 layout); register them as packages explicitly so that
    # this repo's same-named import shims (regular packages, which would win over namespace packages) cannot be picked up
    for pkg in ("nets", "utils", "data"):
        m = types.ModuleType(pkg)
        m.__path__ = [os.path.join(REF, pkg)]
        sys.modules[pkg] = m
    import nets.ColorHandPose3DNetwork as ref_net
    import nets.PosePriorNetwork as ref_prior
    import utils.general as ref_general
    import utils.relative_trafo as ref_rel
    for m in (ref_net, ref_prior, ref_general, ref_rel):
        assert os.path.abspath(m.__file__).startswith(os.path.abspath(REF)), m.__file__
    return tfe, ref_net, ref_prior, ref_general, ref_rel


def prior_scoremap():
    """[2,256,256,21] score maps from exact integer arithmetic (not stored in the fixture; the test recomputes them)."""
    b, y, x, c = np.meshgrid(np.arange(2), np.arange(256), np.arange(256), np.arange(21), indexing="ij")
    v = ((b * 11 + y * 37 + x * 101 + c * 53 + (y * x) % 29 * 7) % 97).astype(np.float32)
    return (v / np.float32(97.0) - np.float32(0.5)).astype(np.float32)


def inputs():
    from hand3d_b200 import weights as Wt
    d = {}
    d["image"] = Wt.synthetic_blob_images(2, 48, 64, seed=41)
    d["hand_side"] = np.array([[1.0, 0.0], [0.0, 1.0]], np.float32)            # one left, one right hand (flip path)
    rng = np.random.default_rng(43)
    d["prior_scoremap"] = prior_scoremap()
    d["coords_xyz"] = rng.normal(scale=0.6, size=(3, 21, 3)).astype(np.float32)
    d["coords_rel"] = np.stack([rng.uniform(0.2, 1.5, size=(3, 21)), rng.uniform(-1.2, 1.2, size=(3, 21)),
                                rng.uniform(-1.2, 1.2, size=(3, 21))], -1).astype(np.float32)
    return d


def weight_sets():
    from hand3d_b200 import weights as Wt
    return Wt.synthetic_weights(0, seg_shift=0.15), Wt.synthetic_weights(0, bottleneck=True)


def main():
    tf, ref_net, ref_prior, G, R = setup_imports()
    d = inputs()
    wd, wb = weight_sets()
    a = np.asarray
    out = {"image": d["image"], "hand_side": d["hand_side"], "coords_xyz": d["coords_xyz"], "coords_rel": d["coords_rel"]}
    T = lambda x: tf.constant(x)

    # ---- ColorHandPose3DNetwork.inference (nets/ColorHandPose3DNetwork.py:61-99) and its stages
    tf.set_weights(wd)
    net = ref_net.ColorHandPose3DNetwork()
    hand_scoremap, image_crop, scale_crop, center, kp_scoremap, coord3d = net.inference(T(d["image"]), T(d["hand_side"]), tf.constant(True))
    names = [n for n, _ in tf.requested]
    out["variables_requested"] = np.array(sorted(set(names)))
    out["inf_hand_scoremap"] = a(hand_scoremap); out["inf_scale_crop"] = a(scale_crop); out["inf_center"] = a(center)
    out["inf_coord3d"] = a(coord3d)
    out["inf_image_crop_s"] = a(image_crop)[:, ::8, ::8, :]
    out["inf_image_crop_sum"] = np.array([a(image_crop).astype(np.float64).sum(), np.abs(a(image_crop)).astype(np.float64).sum()])
    out["inf_kp_scoremap_s"] = a(kp_scoremap)[:, 3::16, 5::16, :]
    out["inf_kp_uv"] = np.stack([G.detect_keypoints(a(kp_scoremap)[b]) for b in (0, 1)])
    # stages, called one by one on the same tensors
    mask = G.single_obj_scoremap(hand_scoremap)
    out["st_mask_rows"] = a(mask)[..., 0].sum(2); out["st_mask_cols"] = a(mask)[..., 0].sum(1)
    c2, bb, cs = G.calc_center_bb(mask)
    out["st_center"], out["st_bb"], out["st_crop_size"] = a(c2), a(bb), a(cs)
    fg = tf.reduce_max(tf.nn.softmax(hand_scoremap)[:, :, :, 1:], 3)
    out["st_max_loc"] = a(G.find_max_location(fg))
    empty = tf.constant(np.zeros((1, 16, 24, 1), np.float32))                      # empty mask -> the written fall-backs
    with np.errstate(invalid="ignore"):                                            # inf + (-inf) inside the reference: intended
        ce, _, se = G.calc_center_bb(empty)
    out["st_empty_center"], out["st_empty_size"] = a(ce), a(se)
    tf.set_weights(wd)
    s_list = net.inference_pose2d(image_crop)
    assert len(s_list) == 3
    out["pose_s0_s"] = a(s_list[0])[:, ::2, ::2, :]; out["pose_s2"] = a(s_list[2])
    tf.set_weights(wd)
    seg_list = net.inference_detection(T(d["image"]))
    assert len(seg_list) == 1
    out["det_hand_scoremap_max_abs_diff_vs_inference"] = np.float64(np.abs(a(seg_list[0]) - a(hand_scoremap)).max())
    tf.set_weights(wd)
    k2, crop2, scale2, center2 = net.inference2d(T(d["image"]))                    # note the different tuple order (:101-129)
    out["inf2d_tuple_ok"] = np.array([np.array_equal(a(k2), a(kp_scoremap)), np.array_equal(a(crop2), a(image_crop)),
                                      np.array_equal(a(scale2), a(scale_crop)), np.array_equal(a(center2), a(center))])
    tf.set_weights(wd)
    can = net._inference_pose3d_can(s_list[2], T(d["hand_side"]), tf.constant(True))
    rot = net._inference_viewpoint(s_list[2], T(d["hand_side"]), tf.constant(True))
    out["lift_can"], out["lift_rot"] = a(can), a(rot)

    # ---- PosePriorNetwork variants (nets/PosePriorNetwork.py:59-95)
    for variant in ("direct", "bottleneck", "local", "local_w_xyz_loss", "proposed"):
        tf.set_weights(wb if variant == "bottleneck" else wd)
        p = ref_prior.PosePriorNetwork(variant)
        normed, c3, Rm = p.inference(T(d["prior_scoremap"]), T(d["hand_side"]), tf.constant(True))
        out["prior_%s_normed" % variant] = a(normed); out["prior_%s_coord3d" % variant] = a(c3)
        out["prior_%s_has_R" % variant] = np.array(Rm is not None)
        if Rm is not None:
            out["prior_%s_R" % variant] = a(Rm)

    # ---- utils/relative_trafo.py:176-295
    out["rel_fwd"] = a(R.bone_rel_trafo(T(d["coords_xyz"])))
    out["rel_inv"] = a(R.bone_rel_trafo_inv(T(d["coords_rel"])))
    out["rel_roundtrip"] = a(R.bone_rel_trafo_inv(R.bone_rel_trafo(T(d["coords_xyz"]))))

    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes;", len(out), "arrays;", len(set(names)), "distinct variables requested by the reference")
    for k in sorted(out):
        if out[k].size <= 12:
            print(" ", k, np.asarray(out[k]).tolist())


if __name__ == "__main__":
    main()

"""Golden vectors produced by the UNMODIFIED reference (lmb-freiburg/hand3d) for the part of the hot path that is plain numpy.

TensorFlow 1.3 cannot be installed here, so the TF graph functions of the reference cannot run (DESIGN.md 2: "parity unpinned").
`utils/general.py` however also holds the host-side numpy code of the path -- `detect_keypoints` (:331-344), `trafo_coords`
(:347-357), `EvalUtil` (:522-611) and `calc_auc` (:654-659) -- and the module only needs `import tensorflow` to succeed.  This script
puts an EMPTY stand-in module named `tensorflow` into `sys.modules`, imports the reference file from where it lies
(a checkout of lmb-freiburg/hand3d named by $H3D_REFERENCE, read-only, nothing is copied), runs those functions on seeded inputs and stores inputs + outputs in
`golden_reference_numpy.npz`.  tests/test_reference_numpy_golden.py pins the oracle, the host-side mirror and (on the GPU) the
device kernels against it.

    python tests/golden/make_golden_reference_numpy.py        # H3D_REFERENCE=<checkout of lmb-freiburg/hand3d>
"""
import importlib.util
import os
import sys
import types

import numpy as np

REF = os.environ.get("H3D_REFERENCE", "")   # a checkout of lmb-freiburg/hand3d (needed only to regenerate)
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden_reference_numpy.npz")


def load_reference_general():
    for name in ("tensorflow", "tensorflow.python", "tensorflow.python.pywrap_tensorflow"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["tensorflow"].python = sys.modules["tensorflow.python"]
    sys.modules["tensorflow.python"].pywrap_tensorflow = sys.modules["tensorflow.python.pywrap_tensorflow"]
    spec = importlib.util.spec_from_file_location("_hand3d_reference_general", os.path.join(REF, "utils", "general.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def inputs():
    rng = np.random.default_rng(20240917)
    d = {}
    # detect_keypoints: plain maps, a 4-D input that gets squeezed, and maps with exact ties (first occurrence must win)
    d["dk_maps"] = rng.normal(size=(32, 24, 21)).astype(np.float16).astype(np.float32)
    d["dk_maps4"] = rng.normal(size=(1, 24, 24, 21)).astype(np.float16).astype(np.float32)
    ties = rng.normal(size=(32, 32, 21)).astype(np.float16).astype(np.float32)
    for c in range(21):
        ties[(7 * c) % 32, (3 * c + 5) % 32, c] = 9.0
        ties[(7 * c + 11) % 32, (3 * c + 1) % 32, c] = 9.0       # same value elsewhere
    d["dk_ties"] = ties
    # trafo_coords
    d["tc_kp"] = rng.integers(0, 256, size=(21, 2)).astype(np.float64)
    d["tc_center"] = np.array([[153.5, 120.0]])
    d["tc_scale"] = np.array([[1.7320508]])
    # EvalUtil: 60 samples, 2-D (pixels) and 3-D (metres), random visibility, one key-point never visible
    n = 60
    d["ev2_gt"] = rng.uniform(0, 320, size=(n, 21, 2))
    d["ev2_pred"] = d["ev2_gt"] + rng.normal(scale=6.0, size=(n, 21, 2))
    d["ev2_vis"] = rng.uniform(size=(n, 21)) < 0.8
    d["ev2_vis"][:, 13] = False
    d["ev3_gt"] = rng.normal(scale=0.05, size=(n, 21, 3))
    d["ev3_pred"] = d["ev3_gt"] + rng.normal(scale=0.012, size=(n, 21, 3))
    d["ev3_vis"] = rng.uniform(size=(n, 21)) < 0.9
    d["auc_x"] = np.linspace(20.0, 50.0, 7)
    d["auc_y"] = rng.uniform(0.2, 1.0, size=7)
    return d


def main():
    G = load_reference_general()
    d = inputs()
    out = dict(d)
    out["dk_maps_out"] = G.detect_keypoints(d["dk_maps"])
    out["dk_maps4_out"] = G.detect_keypoints(d["dk_maps4"])
    out["dk_ties_out"] = G.detect_keypoints(d["dk_ties"])
    out["tc_out"] = G.trafo_coords(d["tc_kp"], d["tc_center"], d["tc_scale"], 256)
    for tag, lo, hi, steps in (("ev2", 0.0, 30.0, 20), ("ev3", 0.0, 0.05, 100)):
        ev = G.EvalUtil()
        for i in range(d[tag + "_gt"].shape[0]):
            ev.feed(d[tag + "_gt"][i], d[tag + "_vis"][i], d[tag + "_pred"][i])
        mean, median, auc, curve, thr = ev.get_measures(lo, hi, steps)
        out[tag + "_mean"], out[tag + "_median"], out[tag + "_auc"] = np.float64(mean), np.float64(median), np.float64(auc)
        out[tag + "_curve"], out[tag + "_thr"] = np.asarray(curve), np.asarray(thr)
        out[tag + "_range"] = np.array([lo, hi, steps])
        out[tag + "_pck5"] = np.array([np.nan if ev._get_pck(k, thr[len(thr) // 2]) is None else ev._get_pck(k, thr[len(thr) // 2])
                                       for k in range(21)])
    out["auc_out"] = np.float64(G.calc_auc(d["auc_x"], d["auc_y"]))
    for k in ("dk_maps", "dk_maps4", "dk_ties"):      # values are exactly representable in fp16: store them that way
        out[k] = out[k].astype(np.float16)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes;", len(out), "arrays")


if __name__ == "__main__":
    main()

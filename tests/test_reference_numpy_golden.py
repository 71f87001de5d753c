"""Pins the oracle, the host-side API mirror and the device kernels against outputs of the UNMODIFIED reference.

`tests/golden/golden_reference_numpy.npz` was produced by tests/golden/make_golden_reference_numpy.py, which imports
the reference's utils/general.py (with an empty stand-in for the `tensorflow` import) and runs the reference's own numpy code of
the hot path: detect_keypoints (utils/general.py:331-344), trafo_coords (:347-357), EvalUtil (:522-611), calc_auc (:654-659).
These are the only functions of the path that can execute without TensorFlow 1.3; for them parity is pinned to the reference
itself, bit for bit (indices) / to 1e-12 (float64 arithmetic)."""
import os

import numpy as np
import pytest

from oracle import hand3d_oracle as O

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_reference_numpy.npz"))


def _maps(k):
    return G[k].astype(np.float32)


# ------------------------------------------------------------------------------------------- oracle (CPU)
@pytest.mark.parametrize("k", ["dk_maps", "dk_maps4", "dk_ties"])
def test_oracle_detect_keypoints_matches_reference(k):
    out = O.detect_keypoints(_maps(k))
    assert out.dtype == np.float64 and out.shape == (21, 2)
    np.testing.assert_array_equal(out, G[k + "_out"])


def test_oracle_trafo_coords_matches_reference():
    np.testing.assert_allclose(O.trafo_coords(G["tc_kp"], G["tc_center"], G["tc_scale"], 256), G["tc_out"], rtol=0, atol=1e-12)


def _feed_all(ev, tag):
    for i in range(G[tag + "_gt"].shape[0]):
        ev.feed(G[tag + "_gt"][i], G[tag + "_vis"][i], G[tag + "_pred"][i])
    lo, hi, steps = G[tag + "_range"]
    return ev.get_measures(float(lo), float(hi), int(steps))


def _check_measures(m, tag, tol):
    mean, median, auc, curve, thr = m
    np.testing.assert_allclose(mean, G[tag + "_mean"], rtol=tol)
    np.testing.assert_allclose(median, G[tag + "_median"], rtol=tol)
    np.testing.assert_allclose(auc, G[tag + "_auc"], rtol=tol)
    np.testing.assert_allclose(curve, G[tag + "_curve"], rtol=0, atol=tol)
    np.testing.assert_allclose(thr, G[tag + "_thr"], rtol=0, atol=1e-15)


@pytest.mark.parametrize("tag", ["ev2", "ev3"])
def test_oracle_evalutil_matches_reference(tag):
    _check_measures(_feed_all(O.EvalUtil(), tag), tag, 1e-12)


# ------------------------------------------------------------------------------------------- host-side mirror (CPU parts)
def test_mirror_trafo_coords_matches_reference():
    from hand3d_b200.utils.general import trafo_coords
    np.testing.assert_allclose(trafo_coords(G["tc_kp"], G["tc_center"], G["tc_scale"], 256), G["tc_out"], rtol=0, atol=1e-12)
    assert trafo_coords(G["tc_kp"], G["tc_center"], G["tc_scale"], 256) is not G["tc_kp"]      # the reference copies its input


@pytest.mark.parametrize("tag", ["ev2", "ev3"])
def test_mirror_evalutil_numpy_path_matches_reference(tag):
    from hand3d_b200.utils.general import EvalUtil
    ev = EvalUtil()
    _check_measures(_feed_all(ev, tag), tag, 1e-12)
    thr = G[tag + "_thr"]
    pck = np.array([np.nan if ev._get_pck(k, thr[len(thr) // 2]) is None else ev._get_pck(k, thr[len(thr) // 2]) for k in range(21)])
    np.testing.assert_array_equal(np.isnan(pck), np.isnan(G[tag + "_pck5"]))          # key-point 13 of ev2 never has data
    np.testing.assert_allclose(np.nan_to_num(pck), np.nan_to_num(G[tag + "_pck5"]), rtol=0, atol=1e-12)


def test_calc_auc_formula_matches_reference():
    trapz = getattr(np, "trapezoid", None) or np.trapz
    x, y = G["auc_x"], G["auc_y"]
    np.testing.assert_allclose(trapz(y, x) / trapz(np.ones_like(y), x), G["auc_out"], rtol=1e-12)


# ------------------------------------------------------------------------------------------- device kernels (GPU)
@pytest.mark.gpu
@pytest.mark.parametrize("k", ["dk_maps", "dk_maps4", "dk_ties"])
def test_device_detect_keypoints_matches_reference(k):
    import torch
    from hand3d_b200.utils.general import detect_keypoints
    m = _maps(k)
    np.testing.assert_array_equal(detect_keypoints(m), G[k + "_out"])                 # numpy in -> float64 [21,2] like the reference
    t = torch.from_numpy(m if m.ndim == 4 else m[None]).cuda()
    np.testing.assert_array_equal(detect_keypoints(t).cpu().numpy()[0], G[k + "_out"].astype(np.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("tag", ["ev2", "ev3"])
def test_device_evalutil_matches_reference(tag):
    """Batched feed(): distances computed by the device kernel in fp32 -> measures agree with the reference's float64 to ~1e-6."""
    import torch
    from hand3d_b200.utils.general import EvalUtil
    ev = EvalUtil()
    ev.feed(torch.from_numpy(G[tag + "_gt"]).cuda(), torch.from_numpy(G[tag + "_vis"]).cuda(), torch.from_numpy(G[tag + "_pred"]).cuda())
    lo, hi, steps = G[tag + "_range"]
    mean, median, auc, curve, thr = ev.get_measures(float(lo), float(hi), int(steps))
    np.testing.assert_allclose(mean, G[tag + "_mean"], rtol=2e-6)
    np.testing.assert_allclose(median, G[tag + "_median"], rtol=2e-6)
    np.testing.assert_allclose(auc, G[tag + "_auc"], rtol=0, atol=2e-3)               # a distance within 1 ulp of a threshold may flip
    np.testing.assert_allclose(curve, G[tag + "_curve"], rtol=0, atol=2e-3)
    assert len(ev.data[13]) == (0 if tag == "ev2" else len(ev.data[13]))

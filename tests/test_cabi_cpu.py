"""CPU-side checks of the boundary: the library loads without a GPU, exports every symbol that
include/hand3d_b200.h declares, and refuses to compute (loudly) when no sm_90a device is present."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from hand3d_b200 import _lib
    return _lib.load()


def _declared():
    txt = open(os.path.join(ROOT, "include", "hand3d_b200.h")).read()
    return sorted(set(re.findall(r"H3D_API\s+[\w\s\*]+?\b(h3d_\w+)\s*\(", txt)))


def test_header_symbols_all_exported_and_bound(lib):
    from hand3d_b200 import _lib
    names = _declared()
    assert len(names) >= 26
    for n in names:
        assert hasattr(lib, n), "library does not export %s" % n
        assert n in _lib.SIGNATURES, "ctypes binding misses %s" % n
    assert sorted(_lib.SIGNATURES) == names


def test_version_and_error_string(lib):
    assert lib.h3d_version() >= 100
    assert isinstance(lib.h3d_last_error(), bytes)


def test_set_tuning_keys(lib):
    """The nine switches that select a real path are accepted (set to their defaults, so no process-wide state changes); the
    switches of an earlier build that selected nothing on sm_90a are unknown keys."""
    from hand3d_b200 import _lib
    live = {"tc_bn": 0, "tc_chunk_kb": 0, "no_side_stream": 0, "no_pool_fusion": 0, "lift_direct": 0, "c3_ffma": 0, "pdl": 1,
            "fc_chain": 1, "no_seg_fusion": 0}
    for key, default in live.items():
        assert lib.h3d_set_tuning(None, key.encode(), default) == _lib.OK, key
    removed = ["tc_2cta", "tc_c64", "tc_c64x2", "tc_pair128", "tc_stack", "tc_exp", "c3_tma", "c64_tma_out", "tc_chain",
               "tc_small_split", "fuse_c1"]
    for key in removed:
        assert lib.h3d_set_tuning(None, key.encode(), 0) == _lib.EINVAL, key
        assert b"unknown key" in lib.h3d_last_error(), key


def test_no_cpu_fallback(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from hand3d_b200 import _lib
    assert lib.h3d_device_available() == 0
    h = C.c_void_p()
    assert lib.h3d_create(C.byref(h), 0) == _lib.ENODEVICE
    assert b"no CPU fallback" in lib.h3d_last_error()
    from hand3d_b200.nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork
    with pytest.raises(RuntimeError):
        ColorHandPose3DNetwork().init(None, weights={})


def test_product_never_imports_oracle():
    bad = []
    for dirpath, _, files in os.walk(os.path.join(ROOT, "hand3d_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f), errors="replace").read()
                if re.search(r"^\s*(from|import)\s+oracle\b", src, re.M):
                    bad.append(f)
    assert not bad, "product files import the oracle: %s" % bad


def test_arch_tables_match_survey():
    from hand3d_b200 import arch
    assert abs(arch.conv_flops_per_image() / 1e9 - 142.258) < 1e-3
    shapes = arch.variable_shapes()
    assert len(shapes) == 134
    assert sum(int(np.prod(s)) for s in shapes.values()) == 34996515


def test_synthetic_weights_and_reference_pickle_layout(tmp_path):
    import pickle
    from hand3d_b200 import weights as Wt
    w = Wt.synthetic_weights(0)
    Wt.validate(w)
    assert w["HandSegNet/conv1_1/weights"].shape == (3, 3, 3, 64) and w["PoseNet2D/conv6_1/weights"].shape == (7, 7, 149, 128)
    assert w["ViewpointNet/fc_vp0/weights"].shape == (4098, 256)
    sub = {k: v for k, v in w.items() if k.startswith("PosePrior/fc")}
    p = tmp_path / "lifting.pickle"
    with open(p, "wb") as f:
        pickle.dump(sub, f, protocol=2)
    back = Wt.load_weight_files([str(p)], exclude_var_list=["fc_xyz"], verbose=False)
    assert set(back) == {k for k in sub if "fc_xyz" not in k}
    with pytest.raises(AssertionError):
        Wt.load_weight_files([str(tmp_path / "missing.pickle")])
    with pytest.raises(ValueError):
        Wt.validate({"Foo/bar/weights": np.zeros(3)})

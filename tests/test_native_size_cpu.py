"""Images above 512 px a side, without a GPU: the pipeline's size limit is declared and bound, and the host grower the GPU tests compare
against (tests/grow_oracle.py) equals the reference's op sequence where the pass budget binds."""
import os
import re

import numpy as np
import pytest

import grow_oracle as G
from hand3d_b200 import _lib
from oracle import hand3d_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_limit_declared_and_bound():
    hdr = open(os.path.join(ROOT, "include", "hand3d_b200.h")).read()
    assert int(re.search(r"#define H3D_PIPELINE_MAX_SIDE (\d+)", hdr).group(1)) == _lib.PIPELINE_MAX_SIDE == 2048
    for name in ("h3d_pipeline_forward", "h3d_seg_postprocess"):
        decl = hdr[:hdr.index(name + "(")]
        assert "H3D_PIPELINE_MAX_SIDE" in decl[decl.rindex("/*"):], name   # the comment above the declaration states the limit
        assert name in _lib.SIGNATURES
    assert _lib.load().h3d_version() >= 107


def test_oracle_bool_grower_equals_literal_where_the_pass_budget_binds():
    """At 530x520 (53 passes) a corridor longer than 530 px is cut by the pass count: the boolean restatement that
    tests/test_gpu_native_size.py compares against must still equal the literal dilation2d / multiply / round sequence."""
    H, W = 530, 520
    logits = G.logits_of([G.make_case(H, W, "serpentine"), G.make_case(H, W, "crossing", 3)])
    lit = O.single_obj_scoremap(logits, literal=True)
    boo = O.single_obj_scoremap(logits, literal=False)
    np.testing.assert_array_equal(lit, boo)
    assert 0 < lit[0].sum() < (G.make_case(H, W, "serpentine")[0]).sum(), "the pass budget must truncate the corridor"


@pytest.mark.parametrize("H,W", [(530, 520), (17, 700), (700, 17), (300, 613)])
def test_fast_grower_equals_oracle(H, W):
    """grow_oracle (axis windows by shifts, bounding-box crop, fixed-point exit) equals oracle.single_obj_scoremap(literal=False)."""
    cases = [G.make_case(H, W, k, seed=i) for i, k in enumerate(G.KINDS)]
    logits = G.logits_of(cases)
    r = G.seg_postprocess(logits)
    mask = O.single_obj_scoremap(logits, literal=False)
    np.testing.assert_array_equal(r["hand_mask"], mask[..., 0].astype(np.uint8))
    center, _, size = O.calc_center_bb(mask)
    np.testing.assert_array_equal(r["center"], center)
    np.testing.assert_array_equal(r["scale_crop"], O.crop_scale(size))
    fg, _ = O.seg_fg_det(logits)
    np.testing.assert_array_equal(r["max_loc"], O.find_max_location(fg))
    for b, (det, seed) in enumerate(cases):
        assert tuple(r["max_loc"][b]) == seed
    assert r["hand_mask"][G.KINDS.index("empty")].sum() == 0 and r["center"][G.KINDS.index("empty")].tolist() == [160.0, 160.0]

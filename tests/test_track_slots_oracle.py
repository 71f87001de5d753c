"""CPU checks of the per-slot re-detection: the selection rule and the staggered schedule (tests/track_slots_oracle.py), FrameRunner's
schedule table, and the new entry's declaration, export and binding."""
import os
import re

import numpy as np
import pytest

import track_slots_oracle as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_selection_is_in_ascending_slot_order():
    n, slots, sel = S.select([0, 1, 0, 1, 1, 0, 0, 1])
    assert n == 4 and slots.tolist() == [1, 3, 4, 7] and sel.tolist() == [0, 1, 0, 1, 1, 0, 0, 1]


def test_selection_limits():
    n, slots, sel = S.select(np.zeros(5, np.int32))
    assert n == 0 and slots.size == 0 and not sel.any()
    n, slots, sel = S.select(np.ones(5, np.int32))               # a fresh state: every slot
    assert n == 5 and slots.tolist() == list(range(5))
    n, slots, _ = S.select(np.zeros(5, np.int32), np.ones(5, np.int32))
    assert n == 5 and slots.tolist() == list(range(5))


def test_force_and_lost_together():
    n, slots, sel = S.select([1, 0, 0, 1, 0], [0, 0, 1, 1, 0])
    assert n == 3 and slots.tolist() == [0, 2, 3] and sel.tolist() == [1, 0, 1, 1, 0]
    # non-zero values of either flag count, not only 1
    assert S.select([0, -3, 0], [7, 0, 0])[1].tolist() == [0, 1]


@pytest.mark.parametrize("B,every", [(1, 1), (3, 2), (32, 5), (32, 32), (5, 8)])
def test_staggered_schedule(B, every):
    masks = np.array([S.redetect_force(B, every, t) for t in range(3 * every)])
    # every slot is forced once in every window of `every` steps, and the load per step differs by at most one slot
    for b in range(B):
        hits = np.flatnonzero(masks[:, b])
        assert np.all(np.diff(hits) == every) and hits[0] < every
    per_step = masks.sum(1)
    assert per_step.max() - per_step.min() <= 1
    assert per_step[:every].sum() == B


def test_frame_runner_schedule_table_matches():
    pytest.importorskip("torch")
    from hand3d_b200.frames import redetect_schedule
    for B, every in [(1, 1), (3, 2), (32, 5), (7, 30)]:
        tab = redetect_schedule(B, every)
        assert tab.dtype == np.int32 and tab.shape == (every, B)
        for t in range(2 * every):
            np.testing.assert_array_equal(tab[t % every], S.redetect_force(B, every, t))


def test_entry_is_declared_bound_and_exported():
    hdr = open(os.path.join(ROOT, "include", "hand3d_b200.h")).read()
    assert re.search(r"H3D_API int h3d_track_step_slots\(", hdr)
    lib = open(os.path.join(ROOT, "hand3d_b200", "_lib.py")).read()
    assert '"h3d_track_step_slots"' in lib
    src = open(os.path.join(ROOT, "hand3d_b200", "csrc", "api.cu")).read()
    assert re.search(r"int h3d_track_step_slots\(", src)
    m = re.search(r"int h3d_version\(void\) \{ return (\d+); \}", src)
    assert m and int(m.group(1)) >= 109
    so = os.path.join(ROOT, "hand3d_b200", "libhand3d_b200.so")
    if not os.path.exists(so):
        pytest.skip("library not built")
    import ctypes
    assert hasattr(ctypes.CDLL(so), "h3d_track_step_slots")

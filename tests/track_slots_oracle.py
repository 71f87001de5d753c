"""numpy restatement of the slot selection of h3d_track_step_slots (DESIGN.md section 4.15) and of the staggered re-detection schedule
of FrameRunner(track=True, detect="slots", redetect_every=N)."""
import numpy as np


def select(lost, force=None):
    """lost, force: int [B] (force may be None) -> (n, slots [n] int32 ascending, selected [B] int32).  Slot b is selected when
    lost[b] != 0 or force[b] != 0."""
    lost = np.asarray(lost)
    sel = lost != 0
    if force is not None:
        sel = sel | (np.asarray(force) != 0)
    slots = np.flatnonzero(sel).astype(np.int32)
    return len(slots), slots, sel.astype(np.int32)


def redetect_force(B, every, t):
    """The force mask of step t: slot b is forced when (t + b) % every == 0."""
    return np.array([int((t + b) % every == 0) for b in range(B)], np.int32)

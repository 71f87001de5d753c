"""Golden record of the UNMODIFIED reference's plot helpers, plot_hand and plot_hand_3d (utils/general.py:360-477).

Both functions only call axis.plot and axis.view_init, so matplotlib is not needed: this script imports the reference's
utils/general.py from where it lies ($H3D_REFERENCE, a read-only checkout of lmb-freiburg/hand3d; nothing is copied) with an empty
stand-in for the `tensorflow` import (as make_golden_reference_numpy.py does), hands them a recording axis on seeded coordinates, and
stores every call's xs, ys (zs), colour and linewidth in golden_reference_plot.npz.  tests/test_reference_plot_golden.py pins
hand3d_b200.draw's BONES, PALETTE and axis order against it.

    python tests/golden/make_golden_reference_plot.py        # H3D_REFERENCE=<checkout of lmb-freiburg/hand3d>
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden_reference_numpy import load_reference_general  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden_reference_plot.npz")
COLOR_FIXED = np.array([0.25, 0.5, 0.75])


class RecordingAxis:
    def __init__(self):
        self.plots, self.views = [], []

    def plot(self, *args, **kwargs):
        arrays = [np.asarray(a, np.float64) for a in args if not (a is COLOR_FIXED)]
        fixed = any(a is COLOR_FIXED for a in args)
        color = COLOR_FIXED if fixed else np.asarray(kwargs["color"], np.float64)
        self.plots.append((arrays, color, fixed, str(kwargs.get("linewidth"))))

    def view_init(self, azim=None, elev=None):
        self.views.append((float(azim), float(elev)))


def _record(out, tag, ax):
    out[tag + "_coords"] = np.stack([np.stack(a, 0) for a, _, _, _ in ax.plots])        # [20, 2 or 3 axes, 2 points]
    out[tag + "_colors"] = np.stack([c for _, c, _, _ in ax.plots])                     # [20, 3]
    out[tag + "_is_fixed"] = np.array([f for _, _, f, _ in ax.plots])
    out[tag + "_linewidth"] = np.array([lw for _, _, _, lw in ax.plots])
    out[tag + "_views"] = np.array(ax.views, np.float64).reshape(-1, 2)                  # (azim, elev)


def main():
    G = load_reference_general()
    rng = np.random.default_rng(20261017)
    out = {"coords_hw": rng.uniform(0, 240, size=(21, 2)), "coords_xyz": rng.normal(size=(21, 3)), "color_fixed": COLOR_FIXED}
    for lw in ("1", "3"):
        for fixed in (False, True):
            tag = "hand_lw%s%s" % (lw, "_fixed" if fixed else "")
            ax = RecordingAxis()
            G.plot_hand(out["coords_hw"], ax, color_fixed=COLOR_FIXED if fixed else None, linewidth=lw)
            _record(out, tag, ax)
            tag = "hand3d_lw%s%s" % (lw, "_fixed" if fixed else "")
            ax = RecordingAxis()
            G.plot_hand_3d(out["coords_xyz"], ax, color_fixed=COLOR_FIXED if fixed else None, linewidth=lw)
            _record(out, tag, ax)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes;", len(out), "arrays")


if __name__ == "__main__":
    main()

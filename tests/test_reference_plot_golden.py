"""Pins hand3d_b200.draw to the UNMODIFIED reference's plot helpers (utils/general.py:360-477), recorded by
tests/golden/make_golden_reference_plot.py: the bones and their order, the jet palette (float32 equality to 255 * c), the axis order
(x = col, y = row for plot_hand; x, y, z for plot_hand_3d), color_fixed, the linewidth and plot_hand_3d's view."""
import os

import numpy as np
import pytest

import draw_oracle as O
from hand3d_b200 import draw as D

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_reference_plot.npz"))
TAGS = ["lw1", "lw1_fixed", "lw3", "lw3_fixed"]


def test_bones_and_order_match_plot_hand():
    hw = G["coords_hw"]
    rec = G["hand_lw1_coords"]                       # [20, (xs, ys), 2 points]
    assert len(D.BONES) == 20 and rec.shape == (20, 2, 2)
    for i, (a, b) in enumerate(D.BONES):
        np.testing.assert_array_equal(rec[i, 0], [hw[a, 1], hw[b, 1]])    # xs = columns
        np.testing.assert_array_equal(rec[i, 1], [hw[a, 0], hw[b, 0]])    # ys = rows


def test_palette_is_255_times_the_reference_colours():
    c = G["hand_lw1_colors"]
    assert D.PALETTE.dtype == np.float32 and D.PALETTE.shape == (20, 3)
    np.testing.assert_array_equal(D.PALETTE, np.float32(255.0 * c))
    np.testing.assert_array_equal(G["hand3d_lw1_colors"], c)             # plot_hand_3d uses the same table
    frac = D.PALETTE - np.floor(D.PALETTE)
    assert {84.5, 248.5} <= set(D.PALETTE[frac == 0.5].tolist())            # kept in float, rounded only after blending


def test_hand_segments_are_the_reference_lines():
    """The oracle's segments (r0, c0, r1, c1) from draw.BONES are exactly the reference's (ys, xs) line end points."""
    seg = O.hand_segments(G["coords_hw"][None].astype(np.float32), D.BONES)[0]
    rec = G["hand_lw1_coords"].astype(np.float32)
    np.testing.assert_array_equal(seg, np.stack([rec[:, 1, 0], rec[:, 0, 0], rec[:, 1, 1], rec[:, 0, 1]], 1))


@pytest.mark.parametrize("tag", TAGS)
def test_calls_colour_and_linewidth(tag):
    fixed = tag.endswith("fixed")
    lw = tag[2]
    for kind in ("hand", "hand3d"):
        assert (G["%s_%s_is_fixed" % (kind, tag)] == fixed).all()
        assert (G["%s_%s_linewidth" % (kind, tag)] == lw).all()
        want = np.repeat(G["color_fixed"][None], 20, 0) if fixed else G["hand_lw1_colors"]
        np.testing.assert_array_equal(G["%s_%s_colors" % (kind, tag)], want)
        np.testing.assert_array_equal(D._colors(G["color_fixed"] if fixed else None), np.float32(255.0 * want))


@pytest.mark.parametrize("tag", TAGS)
def test_plot_hand_3d_axis_order_and_view(tag):
    xyz = G["coords_xyz"]
    rec = G["hand3d_%s_coords" % tag]                # [20, (xs, ys, zs), 2 points]
    for i, (a, b) in enumerate(D.BONES):
        for ax in range(3):
            np.testing.assert_array_equal(rec[i, ax], [xyz[a, ax], xyz[b, ax]])
    np.testing.assert_array_equal(G["hand3d_%s_views" % tag], [[-90.0, 90.0]])
    assert G["hand_%s_views" % tag].shape == (0, 2)                          # plot_hand sets no view

"""run.py's pictures on the device: plot_hand / plot_hand_3d (utils/general.py:360-477) and run.py's four-panel figure (run.py:76-92)
drawn into uint8 RGB images by one CUDA kernel (Context.draw_segments, h3d_draw_segments; DESIGN.md section 4.16).

matplotlib itself (axes, ticks, text, mplot3d's perspective) is not mirrored: what is drawn is the stick figure, the crop square and
the images, pixel for pixel by the rule stated in include/hand3d_b200.h.
"""
from __future__ import annotations

import numpy as np
import torch

from . import runtime
from .utils.general import trafo_coords

# plot_hand's bones, in its drawing order (utils/general.py:384-407): the thumb first, then each finger from the palm outwards
BONES = ((0, 4), (4, 3), (3, 2), (2, 1),
         (0, 8), (8, 7), (7, 6), (6, 5),
         (0, 12), (12, 11), (11, 10), (10, 9),
         (0, 16), (16, 15), (15, 14), (14, 13),
         (0, 20), (20, 19), (19, 18), (18, 17))

# matplotlib's jet colour map as its public segment data: (x, y below x, y above x) per channel
_JET = {"red": ((0., 0, 0), (0.35, 0, 0), (0.66, 1, 1), (0.89, 1, 1), (1, 0.5, 0.5)),
        "green": ((0., 0, 0), (0.125, 0, 0), (0.375, 1, 1), (0.64, 1, 1), (0.91, 0, 0), (1, 0, 0)),
        "blue": ((0., 0.5, 0.5), (0.11, 1, 1), (0.34, 1, 1), (0.65, 0, 0), (1, 0, 0))}


def _segment_lut(data, N=256):
    """LinearSegmentedColormap's N-entry table of one channel (matplotlib's _create_lookup_table with gamma 1)."""
    a = np.asarray(data, np.float64)
    x, y0, y1 = a[:, 0] * (N - 1), a[:, 1], a[:, 2]
    xind = (N - 1) * np.linspace(0, 1, N)
    ind = np.searchsorted(x, xind)[1:-1]
    dist = (xind[1:-1] - x[ind - 1]) / (x[ind] - x[ind - 1])
    return np.clip(np.concatenate([[y1[0]], dist * (y0[ind] - y1[ind - 1]) + y1[ind - 1], [y0[-1]]]), 0.0, 1.0)


def _jet(values, N=256):
    """jet(values) for floats in [0, 1], sampled as Colormap.__call__ samples its table: index int(v * N), with v == 1 -> N - 1."""
    lut = np.stack([_segment_lut(_JET[c], N) for c in ("red", "green", "blue")], 1)
    xa = np.asarray(values, np.float64) * N
    xa[xa == N] = N - 1
    return lut[np.clip(xa, 0, N - 1).astype(int)]


# plot_hand's colours, 255 * jet(linspace(0, 1, 20)) in float32.  Kept in float: two entries are exactly 84.5 and 248.5, so bytes
# would depend on a rounding the reference never makes; the kernel rounds once, after blending.
PALETTE = np.float32(255.0 * _jet(np.linspace(0, 1, len(BONES))))
WHITE = np.float32([255.0, 255.0, 255.0])
# imshow's default colour map (viridis) at its two ends, as Colormap(..., bytes=True) gives them: argmax of the hand score map is 0 or 1
VIRIDIS_ENDS = np.uint8([[68, 1, 84], [253, 231, 36]])
PANEL_3D = (240, 360)   # draw_hand_3d's panel in run_figure: 60 px per unit over run.py's limits x in [-3, 3], y in [-3, 1]

_bone_index = {}


def _bones_on(device):
    """The bones' joint indices as a device tensor [2,20], made once per device (outside any graph capture)."""
    if device not in _bone_index:
        _bone_index[device] = torch.tensor(np.array(BONES).T.copy(), dtype=torch.long, device=device)
    return _bone_index[device]


def _batched_images(images):
    if not isinstance(images, torch.Tensor) or not images.is_cuda or images.dtype != torch.uint8:
        raise TypeError("images must be a CUDA uint8 tensor [B,H,W,3] or [H,W,3]")
    return (images.unsqueeze(0), True) if images.dim() == 3 else (images, False)


def _coords_on(coords, device, n):
    """CUDA or numpy coordinates [B,21,n] (float32 or float64) -> CUDA float32 [B,21,n]."""
    c = torch.from_numpy(np.ascontiguousarray(coords)) if isinstance(coords, np.ndarray) else coords
    c = c.to(device=device, dtype=torch.float32)
    if c.dim() == 2:
        c = c.unsqueeze(0)
    if c.dim() != 3 or c.shape[1] != 21 or c.shape[2] != n:
        raise ValueError("coordinates must be [B,21,%d], got %s" % (n, tuple(c.shape)))
    return c


def _colors(color_fixed):
    if color_fixed is None:
        return PALETTE
    c = np.asarray(color_fixed, np.float64).reshape(3)
    return np.repeat(np.float32(255.0 * c)[None], len(BONES), 0)


def hand_segments(coords_hw):
    """CUDA float32 [B,21,2] (row, col) -> [B,20,4] (r0, c0, r1, c1), plot_hand's bones, by a gather on the device."""
    idx = _bones_on(coords_hw.device)
    return torch.cat([coords_hw[:, idx[0]], coords_hw[:, idx[1]]], -1)


def _valid(valid, B, device):
    if valid is None:
        return None
    v = torch.as_tensor(valid, device=device).reshape(B)
    return v.to(torch.int32) if v.dtype != torch.int32 else v.contiguous()


def draw_hand(images, coords_hw, color_fixed=None, linewidth=1.0, valid=None):
    """plot_hand(coords_hw, axis, color_fixed, linewidth) drawn into images (CUDA uint8 [B,H,W,3] or [H,W,3]) in place; returns them.

    coords_hw [B,21,2] (row, col) in the images' pixels, float32 or float64, CUDA or numpy (rounded to float32).  color_fixed is an RGB
    triple in 0..1 (None: plot_hand's jet colours, PALETTE).  valid [B] (0 = leave image b alone) or None.  With CUDA coordinates the
    call never synchronises the host, so it can be captured into a CUDA graph (once the bone indices exist on the device, i.e. after
    one call outside capture)."""
    imgs, _ = _batched_images(images)
    c = _coords_on(coords_hw, imgs.device, 2)
    ctx = runtime.default_context(imgs.device)
    ctx.draw_segments(imgs, hand_segments(c).contiguous(), _colors(color_fixed), linewidth, _valid(valid, imgs.shape[0], imgs.device))
    return images


def project_3d(coords_xyz, panel_hw, xlim=(-3.0, 3.0), ylim=(-3.0, 1.0)):
    """The orthographic view of draw_hand_3d: CUDA float32 [B,21,3] -> (row, col) [B,21,2] float32, with
    col = (x - xlim[0]) * W / (xlim[1] - xlim[0]) - 0.5 and row = (y - ylim[0]) * H / (ylim[1] - ylim[0]) - 0.5, each step in float32."""
    H, W = panel_hw
    x, y = coords_xyz[..., 0], coords_xyz[..., 1]

    def full(v, like):      # divide by tensors: torch turns a division by a Python scalar into a multiplication by its reciprocal
        return torch.full_like(like, float(np.float32(v)))
    sx = full(np.float32(xlim[1]) - np.float32(xlim[0]), x)
    sy = full(np.float32(ylim[1]) - np.float32(ylim[0]), y)
    cols = (x - full(xlim[0], x)) * full(W, x) / sx - full(0.5, x)
    rows = (y - full(ylim[0], y)) * full(H, y) / sy - full(0.5, y)
    return torch.stack([rows, cols], -1)


def draw_hand_3d(panels, coords_xyz, xlim=(-3.0, 3.0), ylim=(-3.0, 1.0), color_fixed=None, linewidth=1.0, valid=None):
    """run.py's fourth panel (run.py:87-91): plot_hand_3d(coords_xyz, ax4) seen with view_init(azim=-90, elev=-90), which aligns the
    3-D coordinates with the camera view: x grows to the right and y downwards.  panels: CUDA uint8 [B,H,W,3] or [H,W,3], drawn in
    place and returned; coords_xyz [B,21,3].

    This is an orthographic projection along the camera axis onto the window xlim x ylim (project_3d), not mplot3d's perspective
    rendering: z is dropped, and there are no axes, ticks or panes."""
    imgs, _ = _batched_images(panels)
    c = _coords_on(coords_xyz, imgs.device, 3)
    hw = project_3d(c, imgs.shape[1:3], xlim, ylim)
    ctx = runtime.default_context(imgs.device)
    ctx.draw_segments(imgs, hand_segments(hw).contiguous(), _colors(color_fixed), linewidth, _valid(valid, imgs.shape[0], imgs.device))
    return panels


def crop_box_segments(center, scale_crop, frame_hw=None, size=(240, 320)):
    """The four sides of the crop a step used, [B,4,4] float32 (r0, c0, r1, c1): the square of side 256 / scale around center in the
    network image of `size` (what crop_image_from_xy cut and trafo_coords maps back from), computed in float64 on the device and
    mapped to frame pixels by frames.frame_coords(corners, frame_hw, size) when frame_hw is given.  Nothing synchronises the host
    (capturable)."""
    from .frames import frame_coords
    c = center.to(torch.float64).reshape(-1, 2)
    s = scale_crop.to(torch.float64).reshape(-1)
    half = torch.full_like(s, 128.0) / s
    r0, r1 = c[:, 0] - half, c[:, 0] + half
    c0, c1 = c[:, 1] - half, c[:, 1] + half
    corners = torch.stack([torch.stack([r0, c0], -1), torch.stack([r0, c1], -1), torch.stack([r1, c1], -1), torch.stack([r1, c0], -1)], 1)
    if frame_hw is not None:
        corners = frame_coords(corners, frame_hw, size)
    return torch.cat([corners, torch.roll(corners, -1, 1)], -1).to(torch.float32)


def crop_panel(image_crop):
    """run.py:72, ((image_crop + 0.5) * 255).astype('uint8'), in float32 on the device: CUDA [B,256,256,3] -> uint8, truncated after
    clamping to 0..255 (numpy's cast of values outside that range is platform-defined)."""
    v = (image_crop + 0.5) * 255.0
    return v.clamp_(0.0, 255.0).to(torch.uint8)


def mask_panel(hand_scoremap):
    """run.py:86, imshow(argmax(hand_scoremap, 2)) with imshow's defaults: [B,H,W,2] -> uint8 [B,H,W,3] in viridis' two ends (ties
    give 0, np.argmax's first maximum)."""
    hand = hand_scoremap[..., 1] > hand_scoremap[..., 0]
    ends = torch.from_numpy(VIRIDIS_ENDS).to(hand_scoremap.device)
    return ends[hand.to(torch.long)]


def run_figure(image_u8, result, linewidth=1.0):
    """run.py's figure (run.py:76-92) for a batch: image_u8 CUDA uint8 [B,240,320,3] (or [240,320,3]), the imresized network image,
    and `result`, Context.pipeline's outputs="all" dict for it.  Returns a dict of uint8 CUDA tensors:
      image [B,240,320,3]   panel 221, the image with plot_hand at trafo_coords of the key-points;
      crop [B,256,256,3]    panel 222, ((crop + 0.5) * 255).astype(uint8) with plot_hand at the crop's key-points;
      mask [B,240,320,3]    panel 223, argmax of the hand score map (mask_panel);
      pose3d [B,240,360,3]  panel 224, draw_hand_3d on a white panel;
      grid [B,512,720,3]    the four in a 2x2 grid of 256x360 cells, each panel centred on white."""
    imgs, squeeze = _batched_images(image_u8)
    uv = result["keypoints_uv"]
    coord_hw = trafo_coords(uv, result["center"], result["scale_crop"], 256)
    p1 = draw_hand(imgs.clone(), coord_hw, linewidth=linewidth)
    p2 = draw_hand(crop_panel(result["image_crop"]).contiguous(), uv, linewidth=linewidth)
    p3 = mask_panel(result["hand_scoremap"]).contiguous()
    B = imgs.shape[0]
    p4 = torch.full((B,) + PANEL_3D + (3,), 255, dtype=torch.uint8, device=imgs.device)
    draw_hand_3d(p4, result["keypoint_coord3d"], linewidth=linewidth)
    ch, cw = 256, 360
    grid = torch.full((B, 2 * ch, 2 * cw, 3), 255, dtype=torch.uint8, device=imgs.device)
    for i, p in enumerate((p1, p2, p3, p4)):
        r, c = divmod(i, 2)
        h, w = p.shape[1:3]
        y, x = r * ch + (ch - h) // 2, c * cw + (cw - w) // 2
        grid[:, y:y + h, x:x + w] = p
    out = {"image": p1, "crop": p2, "mask": p3, "pose3d": p4, "grid": grid}
    return {k: v[0] for k, v in out.items()} if squeeze else out

"""numpy float32 restatement of h3d_draw_segments (include/hand3d_b200.h, DESIGN.md section 4.16): anti-aliased segments drawn
into uint8 RGB images, later segments over earlier ones.

Each segment reaches only the pixels of its end points' box expanded by g = h + 1 (in float32, clipped to the image), as the rule
states.  For end points within 2^14 px of the image that box changes nothing (d > h outside it after rounding too):
test_draw_oracle.py checks the windows against the box-free evaluation (full=True) there, and shows where they part farther out."""
import numpy as np

F = np.float32


def _clamp01(v):
    """min(max(v, 0), 1) with NaN -> 0, as the kernel's comparisons give it."""
    return np.where(v > F(0), np.where(v < F(1), v, F(1)), F(0)).astype(F)


def coverage(ys, xs, seg, h):
    """Coverage a of pixels (ys, xs) (float32 grids) by one finite segment (r0, c0, r1, c1), in the rule's order."""
    r0, c0, r1, c1 = (F(v) for v in seg)
    with np.errstate(all="ignore"):
        dy, dx = F(r1 - r0), F(c1 - c0)
        L2 = F(F(dy * dy) + F(dx * dx))
        ry, rx = (ys - r0).astype(F), (xs - c0).astype(F)
        num = (ry * dy).astype(F) + (rx * dx).astype(F)
        t = _clamp01((num / L2).astype(F)) if L2 > 0 else np.zeros_like(ry)
        ey = (ry - (t * dy).astype(F)).astype(F)
        ex = (rx - (t * dx).astype(F)).astype(F)
        d = np.sqrt((ey * ey).astype(F) + (ex * ex).astype(F)).astype(F)
        return _clamp01((F(h) - d).astype(F))


def half_width(linewidth):
    return F(F(linewidth) / F(2) + F(0.5))


def draw_image(img, segments, colors, linewidth, full=False):
    """img uint8 [H,W,3] (returned as a new array), segments [S,4], colors [S,3] (0..255)."""
    H, W, _ = img.shape
    h = half_width(linewidth)
    g = F(h + F(1))
    v = img.astype(F)
    touched = np.zeros((H, W), bool)
    segments = np.asarray(segments, F)
    colors = np.asarray(colors, F)
    for k in range(segments.shape[0]):
        s = segments[k]
        if not np.isfinite(s).all():
            continue
        if full:
            ylo, yhi, xlo, xhi = 0, H - 1, 0, W - 1
        else:
            with np.errstate(over="ignore"):
                lo_r, hi_r = F(min(s[0], s[2]) - g), F(max(s[0], s[2]) + g)
                lo_c, hi_c = F(min(s[1], s[3]) - g), F(max(s[1], s[3]) + g)
            if hi_r < 0 or lo_r > H - 1 or hi_c < 0 or lo_c > W - 1:
                continue
            ylo, yhi = int(max(np.ceil(lo_r), 0)), int(min(np.floor(hi_r), H - 1))
            xlo, xhi = int(max(np.ceil(lo_c), 0)), int(min(np.floor(hi_c), W - 1))
            if ylo > yhi or xlo > xhi:
                continue
        ys, xs = np.meshgrid(np.arange(ylo, yhi + 1, dtype=F), np.arange(xlo, xhi + 1, dtype=F), indexing="ij")
        a = coverage(ys, xs, s, h)
        on = a > 0
        if not on.any():
            continue
        win = v[ylo:yhi + 1, xlo:xhi + 1]
        for c in range(3):
            ch = win[..., c]
            ch[on] = (ch[on] + (a[on] * (colors[k, c] - ch[on]).astype(F)).astype(F)).astype(F)
        touched[ylo:yhi + 1, xlo:xhi + 1] |= on
    out = img.copy()
    out[touched] = np.clip(np.rint(v[touched]), 0, 255).astype(np.uint8)
    return out


def draw(images, segments, colors, linewidth, valid=None, full=False):
    """images uint8 [B,H,W,3], segments [B,S,4], colors [S,3], valid [B] or None -> the drawn images (new array)."""
    out = np.array(images, copy=True)
    for b in range(out.shape[0]):
        if valid is not None and valid[b] == 0:
            continue
        out[b] = draw_image(out[b], segments[b], colors, linewidth, full)
    return out


def hand_segments(coords_hw, bones):
    """[B,21,2] (row, col) -> [B,len(bones),4] float32 (r0, c0, r1, c1): plot_hand's bones."""
    c = np.asarray(coords_hw).astype(F)
    i = np.array([a for a, _ in bones]), np.array([b for _, b in bones])
    return np.concatenate([c[:, i[0]], c[:, i[1]]], -1)


def project_3d(coords_xyz, H, W, xlim=(-3.0, 3.0), ylim=(-3.0, 1.0)):
    """draw_hand_3d's orthographic view along the camera axis: [B,21,3] -> (row, col) [B,21,2] float32."""
    c = np.asarray(coords_xyz, F)
    with np.errstate(all="ignore"):
        cols = (((c[..., 0] - F(xlim[0])) * F(W)).astype(F) / F(F(xlim[1]) - F(xlim[0]))).astype(F) - F(0.5)
        rows = (((c[..., 1] - F(ylim[0])) * F(H)).astype(F) / F(F(ylim[1]) - F(ylim[0]))).astype(F) - F(0.5)
    return np.stack([rows.astype(F), cols.astype(F)], -1)


def crop_box(center, scale_crop, frame_hw=None, size=(240, 320)):
    """The crop square's four sides [B,4,4] float32: side 256 / scale around center (float64), mapped to frame pixels with Pillow's
    pixel-centre convention when frame_hw is given (frames.frame_coords)."""
    c = np.asarray(center, np.float64).reshape(-1, 2)
    half = 128.0 / np.asarray(scale_crop, np.float64).reshape(-1)
    r0, r1 = c[:, 0] - half, c[:, 0] + half
    c0, c1 = c[:, 1] - half, c[:, 1] + half
    corners = np.stack([np.stack([r0, c0], -1), np.stack([r0, c1], -1), np.stack([r1, c1], -1), np.stack([r1, c0], -1)], 1)
    if frame_hw is not None:
        rows = (corners[..., 0] + 0.5) * float(frame_hw[0]) / float(size[0]) - 0.5
        cols = (corners[..., 1] + 0.5) * float(frame_hw[1]) / float(size[1]) - 0.5
        corners = np.stack([rows, cols], -1)
    nxt = np.roll(corners, -1, axis=1)
    return np.concatenate([corners, nxt], -1).astype(F)

"""single_obj_scoremap + calc_center_bb + the crop scale (utils/general.py:233-328, nets/ColorHandPose3DNetwork.py:83-85) for maps of
up to 2048 px a side, fast enough to check every case of tests/test_gpu_native_size.py on the host.

It is oracle.single_obj_scoremap(literal=False) with three changes that leave the result as it is (test_native_size_cpu.py pins that):
  * the 21x21 box dilation is separable and each axis is a window of 21 built from shifts of 1, 2, 4 and 3 pixels (3, 7, 15, 21);
  * the passes run on the bounding box of det and the seed only: outside it det is 0, so obj is 0 there after the first pass;
  * the loop stops at a fixed point: obj <- det & dilate(obj) changes nothing once it has changed nothing.
"""
import numpy as np

from oracle import hand3d_oracle as O


def _widen(a, axis):
    for s in (1, 2, 4, 3):
        b = a.copy()
        if axis == 1:
            b[:, s:] |= a[:, :-s]
            b[:, :-s] |= a[:, s:]
        else:
            b[s:] |= a[:-s]
            b[:-s] |= a[s:]
        a = b
    return a


def grow(det, seed, num_passes):
    """det [H,W] bool, seed (row, col) -> the object mask [H,W] bool after num_passes passes."""
    H, W = det.shape
    sy, sx = int(seed[0]), int(seed[1])
    rows, cols = np.nonzero(det)
    y0, y1 = min(rows.min(initial=sy), sy), max(rows.max(initial=sy), sy) + 1
    x0, x1 = min(cols.min(initial=sx), sx), max(cols.max(initial=sx), sx) + 1
    d = det[y0:y1, x0:x1]
    o = np.zeros_like(d)
    o[sy - y0, sx - x0] = True
    for _ in range(num_passes):
        n = d & _widen(_widen(o, 1), 0)
        if np.array_equal(n, o):
            break
        o = n
    out = np.zeros((H, W), bool)
    out[y0:y1, x0:x1] = o
    return out


def band_starts(H):
    """First rows of the row bands the cluster grower splits an H-row map into (1..8 bands of >= 16 rows, sizes differing by <= 1)."""
    cs = max(1, min(8, H // 16))
    return [r * (H // cs) + min(r, H % cs) for r in range(cs)]


KINDS = ["blobs", "serpentine", "crossing", "empty", "full", "seed_first_row", "seed_last_row"]


def make_case(H, W, kind, seed=0):
    """Synthetic det mask [H,W] bool and seed pixel of one case kind:
      blobs: random discs; the seed is a disc centre;
      serpentine: a 1-px corridor of rows 11 apart (one more than a pass can jump) joined at alternate ends, seeded at its start, far
        longer than max(H, W) // 10 passes grow, so the pass count truncates the mask;
      crossing: full-width rows at every band boundary b + d, d in (-11, -10, -9, -1, 0, 1, 9, 10, 11), plus sparse random dots that
        percolate through jumps of up to 10 px in every direction;
      empty: no pixel is hand (the fall-backs); full: every pixel is, seeded in the last row's last pixel;
      seed_first_row / seed_last_row: blobs with the seed on the first / last row."""
    rng = np.random.default_rng(seed)
    det = np.zeros((H, W), bool)
    yy, xx = np.mgrid[0:H, 0:W]

    def discs(n):
        c = []
        for _ in range(n):
            cy, cx, r = rng.integers(0, H), rng.integers(0, W), rng.integers(3, max(4, min(H, W) // 6))
            det[(yy - cy) ** 2 + (xx - cx) ** 2 <= r * r] = True
            c.append((cy, cx))
        return c

    if kind == "blobs":
        sy, sx = discs(int(rng.integers(2, 7)))[0]
    elif kind == "serpentine":
        rows = list(range(0, H, 11))
        for i, r in enumerate(rows):
            det[r, :] = True
            if i + 1 < len(rows):
                det[r:rows[i + 1] + 1, W - 1 if i % 2 == 0 else 0] = True
        sy, sx = 0, 0
    elif kind == "crossing":
        for b in band_starts(H)[1:]:
            for d in (-11, -10, -9, -1, 0, 1, 9, 10, 11):
                if 0 <= b + d < H:
                    det[b + d, ::3] = True
        det |= rng.random((H, W)) < 1.0 / 120
        ys, xs = np.nonzero(det)
        sy, sx = ys[0], xs[0]
    elif kind == "empty":
        sy, sx = 0, 0
    elif kind == "full":
        det[:] = True
        sy, sx = H - 1, W - 1
    elif kind in ("seed_first_row", "seed_last_row"):
        discs(3)
        sy = 0 if kind == "seed_first_row" else H - 1
        sx = int(rng.integers(0, W))
        det[sy, max(0, sx - 40):sx + 40] = True
    else:
        raise ValueError(kind)
    return det, (int(sy), int(sx))


def logits_of(cases):
    """[(det, seed)] of one shape -> logits [B,H,W,2] float32: hand pixels +1, others -1, the seed +2 (or -0.5 when it is not hand), so
    that it is the unique arg-max of the hand probability."""
    H, W = cases[0][0].shape
    out = np.zeros((len(cases), H, W, 2), np.float32)
    for b, (det, (sy, sx)) in enumerate(cases):
        out[b, ..., 1] = np.where(det, 1.0, -1.0)
        out[b, sy, sx, 1] = 2.0 if det[sy, sx] else -0.5
    return out


def seg_postprocess(logits):
    """logits [B,H,W,2] float32 -> dict of hand_mask [B,H,W] uint8, max_loc [B,2] int32, center [B,2], crop_size [B,1], scale_crop [B,1],
    as Context.seg_postprocess returns them."""
    B, H, W, _ = logits.shape
    fg, det = O.seg_fg_det(logits)
    loc = O.find_max_location(fg)
    passes = max(H, W) // (21 // 2)
    mask = np.stack([grow(det[b] > 0.5, loc[b], passes) for b in range(B)]).astype(np.uint8)
    center, _, size = O.calc_center_bb(mask)
    return {"hand_mask": mask, "max_loc": loc, "center": center, "crop_size": size, "scale_crop": O.crop_scale(size)}

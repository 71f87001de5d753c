"""numpy restatement of scipy.misc.imresize(frame, (h, w)) with interp='bilinear' (run.py:57-59), i.e. Pillow's 8-bit BILINEAR
resample (libImaging/Resample.c), and of run.py's normalisation.  Test-only: it is the yardstick of hand3d_b200.frames."""
import hashlib

import numpy as np

PRECISION_BITS = 22   # 32 - 8 - 2
GOLDEN_ROW_STEP = 16  # golden_frames_pil.npz keeps every 16th output row in full, beside the digest of the whole output


def coeffs(in_size, out_size):
    """Pillow's precompute_coeffs + normalize_coeffs_8bpc for the triangle filter -> ([(first tap, taps)], int64 [out, ksize])."""
    scale = in_size / out_size
    filterscale = max(scale, 1.0)
    support = 1.0 * filterscale
    ksize = int(np.ceil(support)) * 2 + 1
    ss = 1.0 / filterscale
    bounds, kk = [], np.zeros((out_size, ksize), np.int64)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [max(0.0, 1.0 - abs((x + xmin - center + 0.5) * ss)) for x in range(xmax)]
        ww = 0.0
        for v in w:                       # sequential double sum, as the C loop
            ww += v
        w = np.array(w) / ww if ww != 0.0 else np.array(w)
        kk[xx, :xmax] = np.where(w < 0, (-0.5 + w * (1 << PRECISION_BITS)).astype(np.int64),
                                 (0.5 + w * (1 << PRECISION_BITS)).astype(np.int64))
        bounds.append((xmin, xmax))
    return bounds, kk


def _pass(a, axis, out_size):
    a = np.moveaxis(a, axis, 0)
    bounds, kk = coeffs(a.shape[0], out_size)
    out = np.empty((out_size,) + a.shape[1:], np.uint8)
    for i, (xmin, n) in enumerate(bounds):
        acc = np.full(a.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
        for t in range(n):
            acc += a[xmin + t].astype(np.int64) * kk[i, t]
        out[i] = np.clip(acc >> PRECISION_BITS, 0, 255)
    return np.moveaxis(out, 0, axis)


def imresize(frame, h, w):
    """uint8 [H, W, 3] -> uint8 [h, w, 3]: the horizontal pass first (into uint8), then the vertical; an axis that keeps its size
    gets no pass."""
    H, W = frame.shape[:2]
    x = frame
    if W != w:
        x = _pass(x, 1, w)
    if H != h:
        x = _pass(x, 0, h)
    return np.ascontiguousarray(x)


def normalize(u8):
    """run.py:59: image_raw.astype('float') / 255.0 - 0.5, fed to the float32 placeholder."""
    return (u8.astype(np.float64) / 255.0 - 0.5).astype(np.float32)


def frame(seed, H, W):
    """The seeded test frame of the golden file: noise over a colour gradient (so both smooth and sharp content is resampled)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
    base = np.stack([yy * 200, xx * 200, (1 - yy) * 100 + xx * 100], -1)
    return np.clip(base + rng.integers(-24, 25, (H, W, 3)), 0, 255).astype(np.uint8)


def golden_digest(out):
    """SHA-256 of a uint8 [h, w, 3] output's shape and bytes."""
    out = np.ascontiguousarray(out, np.uint8)
    return hashlib.sha256(repr(out.shape).encode() + out.tobytes()).hexdigest()


def assert_equals_golden(out, z, i):
    """out equals case i of golden_frames_pil.npz bit for bit: its stored rows first (they locate a mismatch), then the digest."""
    np.testing.assert_array_equal(out[::GOLDEN_ROW_STEP], z["rows_%d" % i], err_msg="golden case %d, stored rows" % i)
    assert golden_digest(out) == str(z["digest_%d" % i]), "golden case %d: the output differs from Pillow's outside the stored rows" % i


def frame_coords(c, frame_hw, size=(240, 320)):
    """Pillow's pixel-centre mapping of coordinates in the size image to frame pixels: (c + 0.5) * Hf / h - 0.5 (rows), same for
    columns, in float64."""
    c = np.asarray(c, np.float64)
    f = np.array(frame_hw, np.float64)
    s = np.array(size, np.float64)
    return (c + 0.5) * f / s - 0.5

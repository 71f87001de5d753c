"""TEST INFRASTRUCTURE ONLY -- CPU restatement (numpy) of the RHD reader's training mode (data/BinaryDbReader.py:160-401) as the
project implements it (hand3d_b200/csrc/reader_aug.cu, reader.cu, hand3d_b200/data/BinaryDbReader.py):

* Philox4x64-10 on uint64 arrays and the counter layout of include/hand3d_b200.h (key (seed, stream), counter (serial, value id,
  attempt, 0)), pinned to numpy.random.Philox;
* the per-sample parameter generator (final values: px, factors, offsets, keep bits) and its layout;
* TF 1.3 adjust_hue (non-fused): the rgb_to_hsv / hsv_to_rgb functors of colorspace_op.h in fp32, mod(h + (delta + 1), 1) between;
* the noisy hand-crop arithmetic, the score-map dropout and the random_crop window, sample by sample;
* the steady-state shuffle queue.

Pinned to the reference SOURCE by tests/golden/golden_reference_reader_train.npz (the unmodified reader over the eager TF stand-in,
with scripted random ops that return this module's draws).
"""
from __future__ import annotations

import numpy as np

from oracle import hand3d_oracle as O
from oracle import reader_oracle as R

f32 = np.float32
u64 = np.uint64
M64 = (1 << 64) - 1

# include/hand3d_b200.h
STREAM_ITEMS, STREAM_SHUFFLE, MAX_ATTEMPTS = 0, 1, 16
COORD_UV_NOISE, CROP_CENTER_NOISE, CROP_SCALE_NOISE, CROP_OFFSET_NOISE, HUE, RANDOM_CROP, SCOREMAP_DROPOUT = 1, 2, 4, 8, 16, 32, 64
UV_NOISE, CENTER_NOISE, SCALE, OFFSET_NOISE, HUE_DELTA, WINDOW, KEEP, USED, PARAMS = 0, 84, 86, 87, 89, 90, 92, 113, 128
FLAG_NAMES = {"coord_uv_noise": COORD_UV_NOISE, "crop_center_noise": CROP_CENTER_NOISE, "crop_scale_noise": CROP_SCALE_NOISE,
              "crop_offset_noise": CROP_OFFSET_NOISE, "hue_aug": HUE, "random_crop_to_size": RANDOM_CROP, "scoremap_dropout": SCOREMAP_DROPOUT}


def flags_of(**kw):
    return sum(bit for name, bit in FLAG_NAMES.items() if kw.get(name))


# ------------------------------------------------------------------------------------------ Philox4x64-10
_M0, _M1 = u64(0xD2E7470EE14C6C93), u64(0xCA5A826395121157)
_W0, _W1 = u64(0x9E3779B97F4A7C15), u64(0xBB67AE8584CAA73B)
_LO32 = u64(0xFFFFFFFF)


def _mulhilo(a, b):
    a = np.asarray(a, u64)
    al, ah, bl, bh = a & _LO32, a >> u64(32), b & _LO32, b >> u64(32)
    ll, hl, lh, hh = al * bl, ah * bl, al * bh, ah * bh
    cross = (ll >> u64(32)) + (hl & _LO32) + lh
    return hh + (hl >> u64(32)) + (cross >> u64(32)), a * b          # uint64 products wrap mod 2^64


def philox4x64_10(ctr, key):
    """ctr [..., 4], key [..., 2] uint64 -> [..., 4] uint64."""
    with np.errstate(over="ignore"):
        c = [np.array(np.asarray(ctr, u64)[..., i]) for i in range(4)]
        k0, k1 = np.array(np.asarray(key, u64)[..., 0]), np.array(np.asarray(key, u64)[..., 1])
        for r in range(10):
            if r:
                k0, k1 = k0 + _W0, k1 + _W1
            hi0, lo0 = _mulhilo(c[0], _M0)
            hi1, lo1 = _mulhilo(c[2], _M1)
            c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
    return np.stack(c, -1)


def words(seed, serials, vid, attempt=0, stream=STREAM_ITEMS):
    s = np.asarray(serials, u64).reshape(-1)
    ctr = np.stack([s, np.full_like(s, vid), np.full_like(s, attempt), np.zeros_like(s)], -1)
    key = np.broadcast_to(np.array([seed & M64, stream], u64), (s.size, 2))
    return philox4x64_10(ctr, key)


def uniform01(w):
    return (np.asarray(w, u64) >> u64(40)).astype(f32) * f32(2.0 ** -24)


def uniform_range(u, lo, hi):          # TF random_uniform: u * (max - min) + min in fp32
    return (u * (f32(hi) - f32(lo)) + f32(lo)).astype(f32)


def truncated_normal(seed, serials, vid, return_attempts=False):
    """Standard normals on [-2, 2]: Box-Muller (fp64) on (w0, w1) of attempt 0, 1, ...; first accepted of z0, z1, z0', ..."""
    n = np.asarray(serials).size
    out = np.zeros(n, f32)
    used = np.full(n, -1)
    todo = np.ones(n, bool)
    for a in range(MAX_ATTEMPTS):
        w = words(seed, serials, vid, a)
        u1 = ((w[:, 0] >> u64(11)) + u64(1)).astype(np.float64) * 2.0 ** -53
        u2 = (w[:, 1] >> u64(11)).astype(np.float64) * 2.0 ** -53
        r = np.sqrt(-2.0 * np.log(u1))
        for z in ((r * np.cos(2.0 * np.pi * u2)).astype(f32), (r * np.sin(2.0 * np.pi * u2)).astype(f32)):
            ok = todo & (np.abs(z) <= f32(2.0))
            out[ok], used[ok] = z[ok], a
            todo &= ~ok
        if not todo.any():
            break
    return (out, used) if return_attempts else out


def aug_params(seed, serials, flags):
    """h3d_reader_aug_params: [n, PARAMS] fp32 final values; neutral values for the flags that are off."""
    s = np.asarray(serials, np.int64).reshape(-1)
    p = np.zeros((s.size, PARAMS), f32)

    def tn(j, sigma):
        return (truncated_normal(seed, s, j) * f32(sigma) + f32(0.0)).astype(f32)

    if flags & COORD_UV_NOISE:
        for j in range(UV_NOISE, UV_NOISE + 84):
            p[:, j] = tn(j, 2.5)
    if flags & CROP_CENTER_NOISE:
        for j in (CENTER_NOISE, CENTER_NOISE + 1):
            p[:, j] = tn(j, 20.0)
    p[:, SCALE] = uniform_range(uniform01(words(seed, s, SCALE)[:, 0]), 1.0, 1.2) if flags & CROP_SCALE_NOISE else f32(1)
    if flags & CROP_OFFSET_NOISE:
        for j in (OFFSET_NOISE, OFFSET_NOISE + 1):
            p[:, j] = tn(j, 10.0)
    if flags & HUE:
        p[:, HUE_DELTA] = uniform_range(uniform01(words(seed, s, HUE_DELTA)[:, 0]), -0.1, 0.1)
    if flags & RANDOM_CROP:
        for j in (WINDOW, WINDOW + 1):
            p[:, j] = (words(seed, s, j)[:, 0] % u64(65)).astype(f32)
    for j in range(KEEP, KEEP + 21):
        p[:, j] = np.floor(f32(0.8) + uniform01(words(seed, s, j)[:, 0])).astype(f32) if flags & SCOREMAP_DROPOUT else f32(1)
    return p


# ------------------------------------------------------------------------------------------ shuffle queue
def shuffle_words(seed, n):
    """The shuffle stream: word d = Philox((d // 4 + 1, 0, 0, 0), (seed, STREAM_SHUFFLE))[d % 4] (numpy.random.Philox from counter 0)."""
    blocks = (n + 3) // 4
    ctr = np.zeros((blocks, 4), u64)
    ctr[:, 0] = np.arange(1, blocks + 1, dtype=u64)
    key = np.broadcast_to(np.array([seed & M64, STREAM_SHUFFLE], u64), (blocks, 2))
    return philox4x64_10(ctr, key).reshape(-1)[:n]


def shuffle_serials(seed, n, capacity=100):
    """Steady state of shuffle_batch_join(capacity=100, min_after_dequeue=50): a buffer of the next `capacity` stream positions, each
    dequeue takes slot w mod capacity and the stream refills it."""
    slots, nxt, out = list(range(capacity)), capacity, []
    for w in shuffle_words(seed, n):
        k = int(w) % capacity
        out.append(slots[k])
        slots[k], nxt = nxt, nxt + 1
    return np.array(out, np.int64)


# ------------------------------------------------------------------------------------------ adjust_hue (TF 1.3)
def rgb_to_hsv(rgb):
    """colorspace_op.h RGBToHSV in fp32: V = max, range = V - min, S = V > 0 ? range / V : 0, H by the channel holding V."""
    rgb = np.asarray(rgb, f32)
    r, g, b = rgb[..., 0], rgb[..., 1], rgb[..., 2]
    v = np.maximum(np.maximum(r, g), b)
    rng = (v - np.minimum(np.minimum(r, g), b)).astype(f32)
    with np.errstate(divide="ignore", invalid="ignore"):
        s = np.where(v > 0, rng / v, f32(0)).astype(f32)
        norm = ((f32(1) / rng) * f32(1.0 / 6.0)).astype(f32)
        h = np.where(r == v, norm * (g - b), np.where(g == v, norm * (b - r) + f32(2.0 / 6.0), norm * (r - g) + f32(4.0 / 6.0))).astype(f32)
    h = np.where(rng > 0, h, f32(0)).astype(f32)
    h = np.where(h < 0, h + f32(1), h).astype(f32)
    return np.stack([h, s, v], -1)


def hsv_to_rgb(hsv):
    """colorspace_op.h HSVToRGB in fp32."""
    hsv = np.asarray(hsv, f32)
    h, s, v = hsv[..., 0], hsv[..., 1], hsv[..., 2]
    dh = h * f32(6)
    dr = np.clip(np.abs(dh - f32(3)) - f32(1), f32(0), f32(1))
    dg = np.clip(-np.abs(dh - f32(2)) + f32(2), f32(0), f32(1))
    db = np.clip(-np.abs(dh - f32(4)) + f32(2), f32(0), f32(1))
    one_s = -s + f32(1)
    return np.stack([(one_s + s * dr) * v, (one_s + s * dg) * v, (one_s + s * db) * v], -1).astype(f32)


def adjust_hue(image, delta):
    """image_ops_impl.adjust_hue (TF 1.3, TF_ADJUST_HUE_FUSED unset): hue = mod(hue + (delta + 1), 1) between the functors."""
    hsv = rgb_to_hsv(image)
    h = np.fmod(hsv[..., 0] + (f32(delta) + f32(1.0)), f32(1.0)).astype(f32)
    return hsv_to_rgb(np.stack([h, hsv[..., 1], hsv[..., 2]], -1))


def dropout(scoremap, keep, keep_prob=0.8):
    """tf.nn.dropout(x, keep_prob, noise_shape=[1, 1, N]) with the given bits, then the reader's * keep_prob (:362-365)."""
    kp = f32(keep_prob)
    return (((np.asarray(scoremap, f32) / kp) * np.asarray(keep, f32).reshape(1, 1, -1)) * kp).astype(f32)


# ------------------------------------------------------------------------------------------ one training sample
def rhd_items_train(record, params, flags, use_wrist_coord=True, hand_crop=False, scale_to_size=False, sigma=25.0, crop_size=256):
    """BinaryDbReader(mode='training', **flags).get() for ONE record with the draws in params [PARAMS]; with hand_crop, also the
    final crop_center (row, col), which the reader feeds to the crop but does not return."""
    p = np.asarray(params, f32).reshape(-1)
    raw = O.decode_rhd_record(record)
    xyz, uv, vis = raw["keypoint_xyz"].astype(f32), raw["keypoint_uv"].astype(f32), raw["keypoint_vis"].astype(bool)
    if not use_wrist_coord:                                            # :139-162
        xyz = np.concatenate([(f32(0.5) * (xyz[0] + xyz[12]))[None], xyz[1:21], (f32(0.5) * (xyz[21] + xyz[33]))[None], xyz[-20:]], 0)
        uv = np.concatenate([(f32(0.5) * (uv[0] + uv[12]))[None], uv[1:21], (f32(0.5) * (uv[21] + uv[33]))[None], uv[-20:]], 0)
        vis = np.concatenate([[vis[0] | vis[12]], vis[1:21], [vis[21] | vis[33]], vis[-20:]], 0)
    if flags & COORD_UV_NOISE:                                         # :160-164, all 42 before the 21-subset
        uv = (uv + p[UV_NOISE:UV_NOISE + 84].reshape(42, 2)).astype(f32)
    image = raw["image"]
    if flags & HUE:                                                    # :183-184
        image = adjust_hue(image, p[HUE_DELTA])
    parts = raw["hand_parts"]
    d = {"keypoint_xyz": xyz, "keypoint_uv": uv, "cam_mat": raw["cam_mat"], "image": image, "hand_parts": parts,
         "hand_mask": raw["hand_mask"], "keypoint_vis": vis}
    if flags & RANDOM_CROP and not scale_to_size:                      # :382-392
        oy, ox = int(p[WINDOW]), int(p[WINDOW + 1])
        return {"image": image[oy:oy + 256, ox:ox + 256], "hand_parts": parts[oy:oy + 256, ox:ox + 256].astype(np.int32),
                "hand_mask": raw["hand_mask"][oy:oy + 256, ox:ox + 256].astype(np.int32)}
    left = int(((parts > 1) & (parts < 18)).sum()) > int((parts > 17).sum())
    xyz21 = xyz[:21] if left else xyz[-21:]
    d["hand_side"] = np.array([1.0, 0.0] if left else [0.0, 1.0], f32)
    d["keypoint_xyz21"] = xyz21
    rel = xyz21 - xyz21[0]
    scale_len = np.sqrt(np.sum(np.square(rel[12] - rel[11]))).astype(f32)
    d["keypoint_scale"] = scale_len
    d["keypoint_xyz21_normed"] = (rel / scale_len).astype(f32)
    d["keypoint_xyz21_local"] = O.bone_rel_trafo(d["keypoint_xyz21_normed"][None])[0]
    can, rot = R.canonical_trafo(d["keypoint_xyz21_normed"])
    d["keypoint_xyz21_can"] = R.flip_right_hand(can, not left)
    d["rot_mat"] = np.linalg.inv(rot).astype(f32)
    vis21, uv21 = (vis[:21], uv[:21]) if left else (vis[-21:], uv[-21:])
    d["keypoint_vis21"], d["keypoint_uv21"] = vis21, uv21
    size = (320, 320)
    if hand_crop:                                                      # :269-346 with the noises
        center = uv21[12, ::-1].astype(f32)
        if not np.all(np.isfinite(center)):
            center = np.zeros(2, f32)
        if flags & CROP_CENTER_NOISE:
            center = (center + p[CENTER_NOISE:CENTER_NOISE + 2]).astype(f32)
        hw = np.stack([uv21[:, 1][vis21], uv21[:, 0][vis21]], 1)
        mn = np.maximum(hw.min(0) if hw.size else np.full(2, np.inf, f32), f32(0.0))
        mx = np.minimum(hw.max(0) if hw.size else np.full(2, -np.inf, f32), np.array(size, f32))
        best = (f32(2) * np.maximum(mx - center, center - mn)).max()
        best = np.minimum(np.maximum(best, f32(50.0)), f32(500.0))
        if not np.isfinite(best):
            best = f32(200.0)
        scale = f32(np.minimum(np.maximum(f32(crop_size) / f32(best), f32(1.0)), f32(10.0)))
        if flags & CROP_SCALE_NOISE:
            scale = f32(scale * p[SCALE])
        if flags & CROP_OFFSET_NOISE:
            center = (center + p[OFFSET_NOISE:OFFSET_NOISE + 2]).astype(f32)
        d["crop_scale"], d["crop_center"] = scale, center
        d["image_crop"] = O.crop_image_from_xy(image[None], center[None], crop_size, np.array([[scale]], f32))[0]
        u = (uv21[:, 0] - center[1]) * scale + f32(crop_size // 2)
        v = (uv21[:, 1] - center[0]) * scale + f32(crop_size // 2)
        uv21 = np.stack([u, v], 1).astype(f32)
        d["keypoint_uv21"] = uv21
        S = np.array([[scale, 0, 0], [0, scale, 0], [0, 0, 1]], f32)
        t1, t2 = center[0] * scale - f32(crop_size // 2), center[1] * scale - f32(crop_size // 2)
        Tm = np.array([[1, 0, -t2], [0, 1, -t1], [0, 0, 1]], f32)
        d["cam_mat"] = (Tm @ (S @ raw["cam_mat"]).astype(f32)).astype(f32)
        size = (crop_size, crop_size)
    sm = R.create_multiple_gaussian_map(np.stack([uv21[:, 1], uv21[:, 0]], -1), size, sigma, vis21)
    if flags & SCOREMAP_DROPOUT:
        sm = dropout(sm, p[KEEP:KEEP + 21])
    d["scoremap"] = sm
    if scale_to_size:
        from oracle import tf1_ops as T
        img = T.resize_bilinear_tf1(image[None], 240, 320)[0]
        d = {"image": img, "keypoint_uv21": np.stack([d["keypoint_uv21"][:, 0] * f32(1.0), d["keypoint_uv21"][:, 1] * f32(0.75)], 1).astype(f32),
             "keypoint_vis21": d["keypoint_vis21"]}
    return d

"""numpy float32 restatement of the tracking rule of h3d_track_step (DESIGN.md section 4.14): one frame's key-points -> the next
frame's crop, the key-point score and the lost flag, per batch slot.  Every operation is a float32 numpy operation (correctly rounded),
in the kernel's order, so the device must match it bit for bit."""
import numpy as np

F = np.float32
FALLBACK_CENTER, FALLBACK_SIZE = F(160.0), F(100.0)   # calc_center_bb's written fall-backs (utils/general.py:271-328)


def keypoints_image(uv, center, scale):
    """trafo_coords (utils/general.py:347-357) in float32: uv [21,2] int (row, col) in the 256x256 crop -> [21,2]."""
    return (np.asarray(uv).astype(F) - F(128)) / F(scale) + np.asarray(center, F)


def score(map32):
    """map32 [32,32,21] -> (sum_k max of channel k, in k order from +0) / 21; NaN anywhere -> NaN."""
    peaks = np.max(np.asarray(map32, F).reshape(-1, 21), axis=0)
    s = F(0)
    for k in range(21):
        s = F(s + peaks[k])
    return F(s / F(21))


def next_crop(uv, center, scale, margin):
    """-> (center' [2], scale', fallback): the crop calc_center_bb and nets/ColorHandPose3DNetwork.py:82-85 give the key-points."""
    with np.errstate(all="ignore"):                      # x / 0 and inf - inf are part of the rule
        p = keypoints_image(uv, center, scale)
        mx, mn = np.max(p, axis=0), np.min(p, axis=0)    # NaN-propagating, as the kernel's reductions
        c = F(0.5) * (mx + mn)
        ext = mx - mn
        size = F(max(ext[0], ext[1])) if not np.isnan(ext).any() else F(np.nan)
        fallback = not (np.isfinite(c).all() and np.isfinite(size))
        if fallback:
            c, size = np.array([FALLBACK_CENTER, FALLBACK_CENTER], F), FALLBACK_SIZE
        s = np.minimum(np.maximum(F(256) / (size * F(margin)), F(0.25)), F(5.0))
    return c.astype(F), F(s), fallback


def update(state, map32, uv, center, scale, margin, min_score=None):
    """One update of B slots.  state: dict center [B,2], scale [B], score [B], lost [B] (modified in place and returned);
    map32 [B,32,32,21], uv [B,21,2], center [B,2], scale [B] (the step's crop).  A lost slot keeps its state's crop."""
    for b in range(len(uv)):
        c, s, fallback = next_crop(uv[b], center[b], F(np.asarray(scale).reshape(-1)[b]), margin)
        sc = score(map32[b])
        lost = fallback or (min_score is not None and not (sc >= F(min_score)))
        state["score"][b] = sc
        state["lost"][b] = int(lost)
        if not lost:
            state["center"][b] = c
            state["scale"][b] = s
    return state


def new_state(B):
    """The state TrackState starts from: the reference's fall-back crop at its margin 1.25, NaN score, lost."""
    return {"center": np.full((B, 2), 160.0, F), "scale": np.full(B, F(256) / (F(100) * F(1.25)), F),
            "score": np.full(B, np.nan, F), "lost": np.ones(B, np.int32)}

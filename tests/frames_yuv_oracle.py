"""numpy restatement of OpenCV's cvtColor COLOR_YUV2RGB_NV12 / _I420 / _YUYV (BT.601 limited range, 20-bit fixed point, chroma
replicated), the layouts of the camera-frame pixel formats (include/hand3d_b200.h), and their composition with frames_oracle.imresize.
Test-only: it is the yardstick of the pixel formats of hand3d_b200.frames."""
import numpy as np

import frames_oracle as F

FORMATS = ("rgb", "bgr", "nv12", "i420", "yuyv")
YUV_FORMATS = ("nv12", "i420", "yuyv")
CY, CRV, CGV, CGU, CBU = 1220542, 1673527, -852492, -409993, 2116026   # OpenCV's ITUR_BT_601_* coefficients, 20 fractional bits
SHIFT = 20


def frame_shape(fmt, H, W):
    """One H x W frame's array shape in fmt."""
    if fmt in ("nv12", "i420"):
        return (H * 3 // 2, W)
    return (H, W, 2) if fmt == "yuyv" else (H, W, 3)


def picture_hw(fmt, frame):
    """(H, W) of the picture a frame of fmt holds."""
    if fmt in ("nv12", "i420"):
        return frame.shape[0] * 2 // 3, frame.shape[1]
    return frame.shape[0], frame.shape[1]


def planes(fmt, frame):
    """A YUV frame -> (Y [H,W], U, V) with U, V [H/2,W/2] for 4:2:0 and [H,W/2] for YUYV."""
    H, W = picture_hw(fmt, frame)
    if fmt == "yuyv":
        p = frame.reshape(H, W // 2, 4)
        return np.stack([p[..., 0], p[..., 2]], -1).reshape(H, W), p[..., 1], p[..., 3]
    flat = frame.reshape(-1)
    Y = flat[:H * W].reshape(H, W)
    if fmt == "nv12":
        uv = flat[H * W:].reshape(H // 2, W // 2, 2)
        return Y, uv[..., 0], uv[..., 1]
    q = (H // 2) * (W // 2)
    return Y, flat[H * W:H * W + q].reshape(H // 2, W // 2), flat[H * W + q:].reshape(H // 2, W // 2)


def pack(fmt, Y, U, V):
    """planes() inverted: (Y, U, V) -> the frame of fmt (uint8, frame_shape(fmt, H, W))."""
    H, W = Y.shape
    if fmt == "yuyv":
        p = np.stack([Y.reshape(H, W // 2, 2)[..., 0], U, Y.reshape(H, W // 2, 2)[..., 1], V], -1)
        return np.ascontiguousarray(p.reshape(H, W, 2), np.uint8)
    if fmt == "nv12":
        tail = np.stack([U, V], -1).reshape(-1)
    else:
        tail = np.concatenate([U.reshape(-1), V.reshape(-1)])
    return np.concatenate([Y.reshape(-1), tail]).astype(np.uint8).reshape(H * 3 // 2, W)


def yuv_to_rgb(Y, U, V):
    """The conversion rule per pixel: Y [H,W], U and V already replicated to [H,W] -> uint8 [H,W,3]."""
    c = np.maximum(Y.astype(np.int32) - 16, 0) * CY + (1 << (SHIFT - 1))
    u = U.astype(np.int32) - 128
    v = V.astype(np.int32) - 128
    rgb = np.stack([c + CRV * v, c + CGV * v + CGU * u, c + CBU * u], -1) >> SHIFT   # every intermediate fits in int32
    return np.clip(rgb, 0, 255).astype(np.uint8)


def to_rgb(fmt, frame):
    """A frame of fmt -> uint8 RGB [H,W,3]: cvtColor(frame, COLOR_YUV2RGB_*) for the YUV formats, the channels reversed for BGR."""
    if fmt == "rgb":
        return np.ascontiguousarray(frame)
    if fmt == "bgr":
        return np.ascontiguousarray(frame[..., ::-1])
    Y, U, V = planes(fmt, frame)
    ry = 2 if fmt in ("nv12", "i420") else 1
    return yuv_to_rgb(Y, np.repeat(np.repeat(U, ry, 0), 2, 1), np.repeat(np.repeat(V, ry, 0), 2, 1))


def resize(fmt, frame, h, w):
    """Pillow's BILINEAR resize (frames_oracle.imresize) of the frame converted to RGB: what the fused kernel computes."""
    return F.imresize(to_rgb(fmt, frame), h, w)


def random_frame(seed, fmt, H, W):
    """Seeded random bytes in fmt's layout (every code of every plane occurs, clipping included)."""
    return np.random.default_rng(seed).integers(0, 256, frame_shape(fmt, H, W), dtype=np.uint8)


def cv2_code(cv2, fmt):
    """The cvtColor code that converts fmt to RGB."""
    return {"nv12": cv2.COLOR_YUV2RGB_NV12, "i420": cv2.COLOR_YUV2RGB_I420, "yuyv": cv2.COLOR_YUV2RGB_YUYV,
            "bgr": cv2.COLOR_BGR2RGB}[fmt]

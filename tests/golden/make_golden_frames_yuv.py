"""Writes golden_frames_yuv.npz: OpenCV's cvtColor(frame, COLOR_YUV2RGB_NV12 / _I420 / _YUYV) of seeded random frames (the conversion
rule of the camera-frame pixel formats, include/hand3d_b200.h).  Stores the OpenCV version, the seeds and the shapes and, per case, not
the frames but the output's SHA-256 (the whole output, bit for bit) and every GOLDEN_ROW_STEP-th output row in full (so a mismatch shows
where it is), as golden_frames_pil.npz does.

    python tests/golden/make_golden_frames_yuv.py
"""
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from frames_oracle import GOLDEN_ROW_STEP, golden_digest  # noqa: E402
from frames_yuv_oracle import YUV_FORMATS, cv2_code, random_frame  # noqa: E402

# (frame H, W): the smallest frames, even sizes whose halves are odd, and a wide one (random bytes do not compress: the file stays small
# only if the stored rows do)
SIZES = [(2, 2), (4, 6), (66, 90), (242, 322), (128, 1024)]
CASES = [(f, H, W) for f in YUV_FORMATS for H, W in SIZES]


def seed_of(i):
    return 9100 + i


def main():
    out = {"opencv_version": np.array(cv2.__version__), "formats": np.array([c[0] for c in CASES]),
           "sizes": np.array([c[1:] for c in CASES], np.int64), "seeds": np.array([seed_of(i) for i in range(len(CASES))], np.int64)}
    for i, (fmt, H, W) in enumerate(CASES):
        o = cv2.cvtColor(random_frame(seed_of(i), fmt, H, W), cv2_code(cv2, fmt))
        out["digest_%d" % i] = np.array(golden_digest(o))
        out["rows_%d" % i] = o[::GOLDEN_ROW_STEP]
    path = os.path.join(HERE, "golden_frames_yuv.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes, OpenCV", cv2.__version__)


if __name__ == "__main__":
    main()

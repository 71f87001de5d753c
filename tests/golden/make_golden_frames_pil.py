"""Writes golden_frames_pil.npz: Pillow's Image.resize(..., BILINEAR) of the seeded frames of tests/frames_oracle.frame, the bytes
scipy.misc.imresize(frame, (h, w)) returns (run.py:57-59).  Stores the Pillow version and, per case, not the frames but the output's
SHA-256 (the whole output, bit for bit) and every GOLDEN_ROW_STEP-th output row in full (so a mismatch shows where it is).

    python tests/golden/make_golden_frames_pil.py
"""
import os
import sys

import numpy as np
import PIL
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from frames_oracle import GOLDEN_ROW_STEP, frame, golden_digest  # noqa: E402

# (frame H, W, output h, w): shrinking by integer and non-integer factors, enlarging, identity, 1-pixel and prime sizes
CASES = [(1080, 1920, 240, 320), (2160, 3840, 256, 256), (480, 640, 320, 320), (720, 1280, 240, 320), (241, 321, 240, 320),
         (100, 77, 256, 256), (3, 5, 240, 320), (240, 320, 240, 320), (1, 1, 240, 320), (2, 700, 240, 320), (1080, 1920, 1, 7)]


def seed_of(i):
    return 7000 + i


def main():
    out = {"pillow_version": np.array(PIL.__version__), "cases": np.array(CASES, np.int64)}
    for i, (H, W, h, w) in enumerate(CASES):
        o = np.asarray(Image.fromarray(frame(seed_of(i), H, W)).resize((w, h), Image.BILINEAR))
        out["digest_%d" % i] = np.array(golden_digest(o))
        out["rows_%d" % i] = o[::GOLDEN_ROW_STEP]
    path = os.path.join(HERE, "golden_frames_pil.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes, Pillow", PIL.__version__)


if __name__ == "__main__":
    main()

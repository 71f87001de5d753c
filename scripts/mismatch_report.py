#!/usr/bin/env python
"""Free-running / teacher-forced mismatch rates of the CUDA pipeline against the CPU oracle over 64 images per precision mode
(BASELINE.json: key-point indices bit-exact, fp32 outputs within 1e-3, fp16 path within 1e-2).  Needs the GPU:
    python scripts/mismatch_report.py > mismatch.json"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import parity_stats as PS  # noqa: E402
from hand3d_b200 import runtime, weights as Wt  # noqa: E402
from oracle import hand3d_oracle as O  # noqa: E402


def main():
    n = int(os.environ.get("N_IMAGES", "64"))
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    wd = Wt.synthetic_weights(0)
    img = PS.mixed_images(n, seed=21)
    hs = Wt.synthetic_hand_side(n, seed=22)
    t0 = time.time()
    ref = O.inference(img, hs, wd, literal_mask=False)
    crops = Wt.synthetic_images(32, 256, 256, seed=23)
    ref_map = PS.posenet_reference(crops, wd)
    ctx = runtime.default_context()
    out = {"images": n, "oracle_seconds": time.time() - t0, "image_set": "half seeded noise, half blob images (tests/parity_stats.py)",
           "full_pipeline": [], "posenet_only_batch32": []}
    for prec in ("bf16x3", "fp16x3", "fp16", "fp32_ffma"):
        if prec == "fp32_ffma" and n > 16:
            st = PS.full_pipeline_stats(ctx, img[:16], hs[:16], wd, tuple(r[:16] for r in ref), prec, chunk=8)
        else:
            st = PS.full_pipeline_stats(ctx, img, hs, wd, ref, prec)
        out["full_pipeline"].append(st)
        if prec != "fp32_ffma":
            out["posenet_only_batch32"].append(PS.posenet_stats(ctx, crops, wd, ref_map, prec))
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()

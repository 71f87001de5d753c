"""Stage-wise numerical error of every precision mode against the fp64 twin of the oracle (needs the GPU)."""
import json
import sys

import numpy as np
import torch

from hand3d_b200 import runtime, weights as Wt
from oracle import hand3d_oracle as O


def stats(a, ref):
    d = np.abs(a.astype(np.float64) - ref.astype(np.float64))
    return {"max": float(d.max()), "rms": float(np.sqrt((d ** 2).mean())), "ref_rms": float(np.sqrt((ref.astype(np.float64) ** 2).mean())),
            "mean_signed": float((a.astype(np.float64) - ref).mean())}


def main():
    wd = Wt.synthetic_weights(0)
    import os
    nimg = int(os.environ.get("ERR_IMAGES", "2"))
    img = Wt.synthetic_images(nimg, 320, 320, seed=1)
    crop = Wt.synthetic_images(nimg, 256, 256, seed=11)
    ref_seg64 = O.inference_detection(img, wd, dtype=np.float64)[-1]
    ref_seg32 = O.inference_detection(img, wd)[-1]
    ref_pose64 = O.inference_pose2d(crop, wd, dtype=np.float64)
    ref_pose32 = O.inference_pose2d(crop, wd)
    out = {"oracle_fp32": {"seg": stats(ref_seg32, ref_seg64), "pose": [stats(a, b) for a, b in zip(ref_pose32, ref_pose64)]}}
    ctx = runtime.default_context()
    ctx.load_weights(wd)
    for prec in sys.argv[1:] or ["fp32_ffma", "bf16x3", "fp16x3", "fp16_f8c", "fp16", "bf16"]:
        ctx.set_precision(prec)
        seg = ctx.handsegnet(torch.from_numpy(img).cuda()).cpu().numpy()
        pose = [p.cpu().numpy() for p in ctx.posenet(torch.from_numpy(crop).cuda())]
        out[prec] = {"seg": stats(seg, ref_seg64), "seg_vs_oracle32": stats(seg, ref_seg32)["max"],
                     "pose": [stats(a, b) for a, b in zip(pose, ref_pose64)],
                     "pose_vs_oracle32": [stats(a, b)["max"] for a, b in zip(pose, ref_pose32)],
                     "mask_flips_vs_fp64": int(((seg[..., 1] > seg[..., 0]) != (ref_seg64[..., 1] > ref_seg64[..., 0])).sum())}
        print(prec, json.dumps(out[prec]), flush=True)
    print("oracle_fp32", json.dumps(out["oracle_fp32"]))
    json.dump(out, sys.stdout, indent=1)


if __name__ == "__main__":
    main()

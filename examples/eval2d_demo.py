#!/usr/bin/env python
"""Evaluation loop in the shape of the reference's eval2d.py (eval2d.py:44-115) on the GPU at batch rate:
binary RHD records -> on-device decode -> inference2d -> detect_keypoints -> trafo_coords -> EvalUtil.

The RHD evaluation set is not available offline; with no arguments the script fabricates records with the exact
on-disk layout (data/BinaryDbReader.py:103-208) from random images / key-points, so the numbers only demonstrate the
plumbing.  Pass --db path/to/rhd_evaluation.bin for the real evaluation.

--device-resident keeps the records and the distances on the GPU (DeviceEvalUtil) with the reference's dtypes (the float64
prediction is not rounded to float32); --graph then replays each batch from one CUDA graph (examples/_eval_loop.py).
"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from data.BinaryDbReader import BinaryDbReader                       # eval2d.py:34
from nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork       # eval2d.py:35
from utils.general import detect_keypoints, trafo_coords             # eval2d.py:36
from hand3d_b200 import runtime
from examples._eval_loop import add_flags, check_flags, evaluate
from examples._synthetic_db import cleanup, db_path


def make_step(net, device_path=False):
    """eval2d.py:58-106 on a batch.  The default path feeds a float32 prediction; device_path keeps the reference's float64 one and
    its rescaling by tensors: u / scale[1], v / scale[0] and both sides / scale2orig_res (all 1 for the reader's 240 x 320 images)."""
    if device_path:
        dev = runtime.default_context().device
        scale = torch.tensor([240.0 / 240, 320.0 / 320], dtype=torch.float64, device=dev)   # eval2d.py:52-53, image already 240 x 320
        scale2orig_res = torch.tensor(1.0, dtype=torch.float64, device=dev)                 # eval2d.py:101-104 (no `resolution`)

    def step(data, util):
        # eval2d.py:50-52 re-applies tf.image.resize_images(data['image'], (240, 320)): the identity on the already scaled image
        keypoints_scoremap, image_crop, scale_crop, center = net.inference2d(data['image'])       # eval2d.py:58
        coord_hw_crop = detect_keypoints(keypoints_scoremap)              # [B,21,2] (row, col) on device (eval2d.py:93)
        coord_hw = trafo_coords(coord_hw_crop, center, scale_crop, 256)   # eval2d.py:94
        if not device_path:
            coord_uv = torch.stack([coord_hw[:, :, 1], coord_hw[:, :, 0]], -1).to(torch.float32)      # eval2d.py:95
            util.feed(data['keypoint_uv21'], data['keypoint_vis21'], coord_uv)                        # eval2d.py:101-106 (scale = 1 here)
            return
        coord_uv = torch.stack([coord_hw[:, :, 1] / scale[1], coord_hw[:, :, 0] / scale[0]], -1)     # eval2d.py:95-99
        util.feed(data['keypoint_uv21'] / scale2orig_res, data['keypoint_vis21'], coord_uv / scale2orig_res)   # eval2d.py:106
    return step


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument("--db", default=None)
    ap.add_argument("--weights", nargs="*", default=None)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--samples", type=int, default=64)
    add_flags(ap)
    args = ap.parse_args()
    check_flags(ap, args)

    path, tmp = db_path(args.db, "rhd", args.samples)
    try:
        # get dataset (eval2d.py:43): the reader scales image and key-points to 240 x 320 itself (scale_to_size)
        dataset = BinaryDbReader(mode='evaluation', shuffle=False, use_wrist_coord=True, scale_to_size=True, batch_size=args.batch, path_to_db=path,
                                 device_resident=args.device_resident)
        net = ColorHandPose3DNetwork()
        if args.weights:
            net.init(None, weight_files=args.weights, exclude_var_list=['PosePrior', 'ViewpointNet'])      # eval2d.py:78-79
        else:
            from hand3d_b200.weights import synthetic_weights
            net.init(None, weights=synthetic_weights(0), exclude_var_list=['PosePrior', 'ViewpointNet'])
        n = min(dataset.num_samples, args.samples) if not args.db else dataset.num_samples
        util = evaluate(dataset, make_step(net, args.device_resident), n, args.batch, args.device_resident, args.graph)
        mean, median, auc, _, _ = util.get_measures(0.0, 30.0, 20)            # eval2d.py:112
        print('Evaluation results (%d samples):' % n)
        print('Average mean EPE: %.3f pixels' % mean)
        print('Average median EPE: %.3f pixels' % median)
        print('Area under curve: %.3f' % auc)
    finally:
        cleanup(tmp)

#!/usr/bin/env python
"""PoseNet-only evaluation in the shape of the reference's eval2d_gt_cropped.py (:36-98) at batch rate: RHD records -> on-device
decode + GT hand crop (BinaryDbReader mirror, hand_crop=True) -> inference_pose2d -> x8 up-sampling -> detect_keypoints -> EvalUtil.

    python examples/eval2d_gt_cropped_demo.py [--db data/bin/rhd_evaluation.bin] [--weights posenet-rhd-stb.pickle]
                                              [--device-resident [--graph]]

--device-resident keeps the records and the distances on the GPU (DeviceEvalUtil) with the reference's dtypes (float64 key-points
divided by the float32 crop scale); --graph then replays each batch from one CUDA graph (examples/_eval_loop.py).
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from data.BinaryDbReader import BinaryDbReader                       # eval2d_gt_cropped.py:28
from nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork       # eval2d_gt_cropped.py:29
from utils.general import detect_keypoints                           # eval2d_gt_cropped.py:30
from hand3d_b200 import runtime
from examples._eval_loop import add_flags, check_flags, evaluate
from examples._synthetic_db import cleanup, db_path


def make_step(net, ctx, device_path=False):
    """eval2d_gt_cropped.py:45-81 on a batch.  The default path feeds a float32 prediction; device_path keeps the reference's float64
    key-points (detect_keypoints returns float64 there) divided by the float32 crop scale."""
    def step(data, util):
        keypoints_scoremap = net.inference_pose2d(data['image_crop'])[-1]                     # :45-46
        s = data['image_crop'].shape
        keypoints_scoremap = ctx.resize_bilinear(keypoints_scoremap, s[1], s[2])               # :49-50
        coord_hw_pred_crop = detect_keypoints(keypoints_scoremap)                              # :78 (device, [B,21,2])
        crop_scale = data['crop_scale'].reshape(-1, 1, 1)
        if not device_path:
            coord_uv_pred_crop = torch.stack([coord_hw_pred_crop[..., 1], coord_hw_pred_crop[..., 0]], -1).to(torch.float32)   # :79
            util.feed(data['keypoint_uv21'] / crop_scale, data['keypoint_vis21'], coord_uv_pred_crop / crop_scale)            # :81
            return
        coord_hw_pred_crop = coord_hw_pred_crop.to(torch.float64)
        coord_uv_pred_crop = torch.stack([coord_hw_pred_crop[..., 1], coord_hw_pred_crop[..., 0]], -1)                        # :79
        util.feed(data['keypoint_uv21'] / crop_scale, data['keypoint_vis21'], coord_uv_pred_crop / crop_scale)                # :81
    return step


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument("--db", default=None)
    ap.add_argument("--weights", nargs="*", default=None)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--samples", type=int, default=32)
    add_flags(ap)
    args = ap.parse_args()
    check_flags(ap, args)

    path, tmp = db_path(args.db, "rhd", args.samples)
    try:
        dataset = BinaryDbReader(mode='evaluation', shuffle=False, hand_crop=True, use_wrist_coord=False, batch_size=args.batch, path_to_db=path,
                                 device_resident=args.device_resident)   # :37
        net = ColorHandPose3DNetwork()
        if args.weights:
            net.init(None, weight_files=args.weights, exclude_var_list=['PosePrior', 'ViewpointNet'])      # :66
        else:
            from hand3d_b200.weights import synthetic_weights
            net.init(None, weights=synthetic_weights(0), exclude_var_list=['PosePrior', 'ViewpointNet'])
        ctx = runtime.default_context()
        n = min(dataset.num_samples, args.samples) if not args.db else dataset.num_samples
        util = evaluate(dataset, make_step(net, ctx, args.device_resident), n, args.batch, args.device_resident, args.graph)
        mean, median, auc, _, _ = util.get_measures(0.0, 30.0, 20)       # :86
        print('Evaluation results:')
        print('Average mean EPE: %.3f pixels' % mean)
        print('Average median EPE: %.3f pixels' % median)
        print('Area under curve: %.3f' % auc)
    finally:
        cleanup(tmp)

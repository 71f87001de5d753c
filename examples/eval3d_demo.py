#!/usr/bin/env python
"""Lifting-only evaluation in the shape of the reference's eval3d.py (eval3d.py:49-101) at batch rate: RHD records -> on-device
decode + GT hand crop + score-map targets (BinaryDbReader mirror) -> PosePriorNetwork.inference -> EvalUtil.

    python examples/eval3d_demo.py [--db data/bin/rhd_evaluation.bin] [--weights lifting-direct.pickle] [--variant direct]
                                   [--device-resident [--graph]]

--device-resident keeps the records and the distances on the GPU (DeviceEvalUtil); --graph then replays each batch from one CUDA
graph (examples/_eval_loop.py).
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from data.BinaryDbReader import BinaryDbReader                       # eval3d.py:38
from nets.PosePriorNetwork import PosePriorNetwork                   # eval3d.py:39
from examples._eval_loop import add_flags, check_flags, evaluate
from examples._synthetic_db import cleanup, db_path


def make_step(net):
    """eval3d.py:60-97 on a batch: float32 prediction and ground truth, every key-point visible."""
    def step(data, util):
        coord3d_pred, _, _ = net.inference(data['scoremap'], data['hand_side'], True)        # eval3d.py:60
        coord3d_pred = coord3d_pred * data['keypoint_scale'].reshape(-1, 1, 1)                # rescale to meters (eval3d.py:91)
        keypoint_xyz21 = data['keypoint_xyz21'] - data['keypoint_xyz21'][:, :1]               # center gt (eval3d.py:94)
        kp_vis = torch.ones_like(keypoint_xyz21[:, :, 0])
        util.feed(keypoint_xyz21, kp_vis, coord3d_pred)                                      # eval3d.py:97
    return step


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument("--db", default=None)
    ap.add_argument("--weights", nargs="*", default=None)
    ap.add_argument("--variant", default="direct", choices=["direct", "bottleneck", "local", "local_w_xyz_loss", "proposed"])
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--samples", type=int, default=32)
    add_flags(ap)
    args = ap.parse_args()
    check_flags(ap, args)

    path, tmp = db_path(args.db, "rhd", args.samples)
    try:
        # get dataset (eval3d.py:50)
        dataset = BinaryDbReader(mode='evaluation', shuffle=False, hand_crop=True, use_wrist_coord=False, batch_size=args.batch, path_to_db=path,
                                 device_resident=args.device_resident)
        net = PosePriorNetwork(args.variant)                             # eval3d.py:56
        if args.weights:
            net.init(None, weight_files=args.weights)                    # eval3d.py:78
        else:
            from hand3d_b200.weights import synthetic_weights
            w = synthetic_weights(0, bottleneck=args.variant == "bottleneck")
            net.init(None, weights={k: v for k, v in w.items() if k.startswith(("PosePrior", "ViewpointNet"))})
        n = min(dataset.num_samples, args.samples) if not args.db else dataset.num_samples
        util = evaluate(dataset, make_step(net), n, args.batch, args.device_resident, args.graph)
        mean, median, auc, _, _ = util.get_measures(0.0, 0.050, 20)      # eval3d.py:103
        print('Evaluation results for %s:' % args.variant)
        print('Average mean EPE: %.3f mm' % (mean * 1000))
        print('Average median EPE: %.3f mm' % (median * 1000))
        print('Area under curve: %.3f' % auc)
    finally:
        cleanup(tmp)

#!/usr/bin/env python
"""Full-pipeline evaluation in the shape of the reference's eval_full.py (eval_full.py:43-99) at batch rate: STB records ->
on-device decode (+ 480x640 -> 240x320: every 2nd pixel under TF1's legacy bilinear kernel) -> inference -> EvalUtil.

    python examples/eval_full_demo.py [--db data/stb/stb_eval.bin] [--weights handsegnet-rhd.pickle posenet3d-rhd-stb.pickle]
                                      [--device-resident [--graph]]

--device-resident keeps the records and the distances on the GPU (DeviceEvalUtil) and also prints eval_full.py's 20-50 mm AUC;
--graph then replays each batch from one CUDA graph (examples/_eval_loop.py).
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from data.BinaryDbReaderSTB import BinaryDbReaderSTB                 # eval_full.py:39
from nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork       # eval_full.py:40
from utils.general import calc_auc                                   # eval_full.py:41
from hand3d_b200 import runtime
from examples._eval_loop import add_flags, check_flags, evaluate
from examples._synthetic_db import cleanup, db_path


def make_step(net, ctx):
    """eval_full.py:50-87 on a batch: float32 prediction and ground truth."""
    def step(data, util):
        image_scaled = ctx.resize_bilinear(data['image'], 240, 320)                          # eval_full.py:50
        _, _, _, _, _, coord3d_pred = net.inference(image_scaled, data['hand_side'], True)   # eval_full.py:57
        coord3d_pred = coord3d_pred * data['keypoint_scale'].reshape(-1, 1, 1)                # rescale to meters (eval_full.py:82)
        keypoint_xyz21 = data['keypoint_xyz21'] - data['keypoint_xyz21'][:, :1]               # center gt (eval_full.py:85)
        util.feed(keypoint_xyz21, data['keypoint_vis21'], coord3d_pred)                      # eval_full.py:87
    return step


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument("--db", default=None)
    ap.add_argument("--weights", nargs="*", default=None)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--samples", type=int, default=16)
    add_flags(ap)
    args = ap.parse_args()
    check_flags(ap, args)

    path, tmp = db_path(args.db, "stb", args.samples)
    try:
        dataset = BinaryDbReaderSTB(mode='evaluation', shuffle=False, use_wrist_coord=False, batch_size=args.batch, path_to_db=path,
                                    device_resident=args.device_resident)   # eval_full.py:45
        net = ColorHandPose3DNetwork()
        if args.weights:
            net.init(None, weight_files=args.weights)                    # eval_full.py:66-67
        else:
            from hand3d_b200.weights import synthetic_weights
            net.init(None, weights=synthetic_weights(0))
        ctx = runtime.default_context()
        n = min(dataset.num_samples, args.samples) if not args.db else dataset.num_samples
        util = evaluate(dataset, make_step(net, ctx), n, args.batch, args.device_resident, args.graph)
        mean, median, auc, pck_curve_all, threshs = util.get_measures(0.0, 0.050, 20)            # eval_full.py:93
        print('Evaluation results')
        print('Average mean EPE: %.3f mm' % (mean * 1000))
        print('Average median EPE: %.3f mm' % (median * 1000))
        print('Area under curve between 0mm - 50mm: %.3f' % auc)
        if args.device_resident:
            # only use subset that lies in 20mm .. 50mm (eval_full.py:98-101)
            pck_curve_all, threshs = pck_curve_all[8:], threshs[8:] * 1000.0
            auc_subset = calc_auc(threshs, pck_curve_all)
            print('Area under curve between 20mm - 50mm: %.3f' % auc_subset)
    finally:
        cleanup(tmp)

#!/usr/bin/env python
"""HandSegNet training in the shape of the reference's training_handsegnet.py (:28-97) on the project's kernels: RHD records ->
on-device decode (BinaryDbReader mirror) -> inference_detection(train=True) -> softmax cross-entropy against the hand mask -> Adam
with TF 1.3 semantics, loss prints every show_loss_freq and pickled snapshots every snapshot_freq iterations.

    python examples/train_handsegnet_demo.py [--db data/bin/rhd_training.bin] [--weights handsegnet.pickle] [--iters 30]

Without --db it trains on a few synthetic records (examples/_synthetic_db.py) and without --weights from synthetic_weights(0): the
TF checkpoint the reference starts from (load_weights_from_snapshot, :73-75) is not read here.  Snapshots are in the reference's
weight-pickle layout (ColorHandPose3DNetwork().init(weight_files=[...]) loads them), not TF checkpoints.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from data.BinaryDbReader import BinaryDbReader                       # training_handsegnet.py:25
from nets.ColorHandPose3DNetwork import ColorHandPose3DNetwork       # training_handsegnet.py:24
from utils.general import LearningRateScheduler                      # training_handsegnet.py:26
from hand3d_b200 import autograd as A, runtime, weights as Wt
from hand3d_b200.optim import Adam
from examples._synthetic_db import cleanup, db_path

# training parameters (training_handsegnet.py:29-34); max_iter is --iters, the frequencies shrink with it for a short demo run
train_para = {'lr': [1e-5, 1e-6, 1e-7],
              'lr_iter': [20000, 30000],
              'max_iter': 40000,
              'show_loss_freq': 1000,
              'snapshot_freq': 5000,
              'snapshot_dir': 'snapshots_handsegnet'}

if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument("--db", default=None)
    ap.add_argument("--weights", nargs="*", default=None)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--show-loss-freq", type=int, default=5)
    ap.add_argument("--snapshot-freq", type=int, default=0, help="0: only the final snapshot")
    ap.add_argument("--snapshot-dir", default=train_para['snapshot_dir'])
    ap.add_argument("--advance-global-step", action="store_true",
                    help="advance the global step so that the learning-rate schedule takes effect (the reference never does)")
    args = ap.parse_args()
    train_para.update(max_iter=args.iters, show_loss_freq=args.show_loss_freq, snapshot_freq=args.snapshot_freq or args.iters + 1,
                      snapshot_dir=args.snapshot_dir)

    path, tmp = db_path(args.db, "rhd", 16)
    try:
        # training_handsegnet.py:37-39 reads with shuffle=True, hue_aug=True and random_crop_to_size=True.  Shuffling and augmentation
        # are refused by the reader mirror (TF's random streams cannot be matched anyway), so this driver reads whole 320x320 images
        # in file order.
        dataset = BinaryDbReader(mode='training', batch_size=8, shuffle=False, path_to_db=path)

        net = ColorHandPose3DNetwork()
        if args.weights:
            net.init(weight_files=args.weights, exclude_var_list=['PosePrior', 'ViewpointNet', 'PoseNet2D'])
        else:
            net.init(weights={k: v for k, v in Wt.synthetic_weights(0).items() if k.startswith('HandSegNet/')})
        ctx = runtime.default_context()
        ctx.set_precision('bf16x3')
        variables = ctx.variables('HandSegNet')

        # Solver (:63-67).  opt.minimize(loss) is called without global_step, so the reference's global step stays 0 and its
        # learning rate stays lr[0] for the whole run; --advance-global-step makes the schedule take effect.
        lr_scheduler = LearningRateScheduler(values=train_para['lr'], steps=train_para['lr_iter'])
        global_step = 0
        opt = Adam(list(variables.values()), lr=lr_scheduler.get_lr(global_step))

        if not os.path.exists(train_para['snapshot_dir']):
            os.mkdir(train_para['snapshot_dir'])
            print('Created snapshot dir:', train_para['snapshot_dir'])

        for i in range(train_para['max_iter']):
            data = dataset.get()
            hand_mask_pred = net.inference_detection(data['image'], train=True)                              # :47
            loss = 0.0
            for pred_item in hand_mask_pred:                                                                  # :56-60
                # the reader's hand_mask is int32 [B,H,W,2]; softmax_cross_entropy_with_logits takes it as float labels
                loss = loss + A.softmax_xent_loss(pred_item, data['hand_mask'].float())
            opt.zero_grad()
            loss.backward()
            opt.set_lr(lr_scheduler.get_lr(global_step))
            opt.step()
            if args.advance_global_step:
                global_step += 1

            if (i % train_para['show_loss_freq']) == 0:
                print('Iteration %d\t Loss %.1e' % (i, float(loss)))
                sys.stdout.flush()

            if (i % train_para['snapshot_freq']) == 0:
                Wt.save_weight_file('%s/model-%d.pickle' % (train_para['snapshot_dir'], i), variables)
                print('Saved a snapshot.')
                sys.stdout.flush()

        print('Training finished. Saving final snapshot.')
        Wt.save_weight_file('%s/model-%d.pickle' % (train_para['snapshot_dir'], train_para['max_iter']), variables)
    finally:
        cleanup(tmp)

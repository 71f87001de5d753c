#!/usr/bin/env python
"""Lifting-stage training in the shape of the reference's training_lifting.py (:28-111) on the project's kernels: RHD records ->
on-device decode + ground-truth hand crop + Gaussian score maps and the 3-D targets (BinaryDbReader mirror) ->
PosePriorNetwork(variant).inference(train=True) -> the variant's MSE loss -> Adam with TF 1.3 semantics, loss prints every
show_loss_freq and pickled snapshots every snapshot_freq iterations.

    python examples/train_lifting_demo.py --variant {direct,bottleneck,local,local_w_xyz_loss,proposed} [--db rhd_training.bin]
                                          [--iters 30] [--augment] [--seed S] [--device-resident [--graph]] [--dropout SEED]

Like the reference, it starts from the initialisers (weights.xavier_weights: Xavier-uniform weights, biases 1e-4; the same
distributions as tf.global_variables_initializer(), not TF's random values), not from a pickle.  Without --db it trains on a few
synthetic records (examples/_synthetic_db.py).  The reference never feeds its `evaluation` placeholder, whose default is True, so
dropout is the identity in its training too; --dropout SEED trains with evaluation=False instead, as the networks' docstrings describe
(dropout after the hidden FC layers, drawn from the context's generator seeded with SEED).  Snapshots are in the reference's
weight-pickle layout (PosePriorNetwork(variant).init(weight_files=[...]) loads them), not TF checkpoints.  --device-resident keeps the records on the GPU;
--graph then captures reading, the step and Adam once after two eager iterations and replays that CUDA graph for every later
iteration.  Both print the losses of the plain run.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from data.BinaryDbReader import BinaryDbReader                       # training_lifting.py:25
from nets.PosePriorNetwork import PosePriorNetwork                   # training_lifting.py:24
from utils.general import LearningRateScheduler                      # training_lifting.py:26
from hand3d_b200 import autograd as A, runtime, weights as Wt
from hand3d_b200.optim import Adam
from hand3d_b200.train_loop import GraphedIteration
from hand3d_b200.utils.relative_trafo import bone_rel_trafo_inv
from examples._synthetic_db import cleanup, db_path

# training parameters (training_lifting.py:36-41); max_iter is --iters, the frequencies shrink with it for a short demo run
train_para = {'lr': [1e-5, 1e-6],
              'lr_iter': [60000],
              'max_iter': 80000,
              'show_loss_freq': 1000,
              'snapshot_freq': 5000,
              'snapshot_dir': 'snapshots_lifting_%s'}

if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument("--variant", default="proposed", choices=["direct", "bottleneck", "local", "local_w_xyz_loss", "proposed"])
    ap.add_argument("--db", default=None)
    ap.add_argument("--seed", type=int, default=0, help="seed of the initialisers and, with --augment, of the reader")
    ap.add_argument("--augment", action="store_true",
                    help="read as training_lifting.py does: shuffled, with the coordinate and the three crop noises")
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--show-loss-freq", type=int, default=5)
    ap.add_argument("--snapshot-freq", type=int, default=0, help="0: only the final snapshot")
    ap.add_argument("--snapshot-dir", default=None)
    ap.add_argument("--advance-global-step", action="store_true",
                    help="advance the global step so that the learning-rate schedule takes effect (the reference never does)")
    ap.add_argument("--device-resident", action="store_true", help="upload the records to the GPU once; get() then runs on the device")
    ap.add_argument("--graph", action="store_true", help="replay each iteration (reading, step, Adam) from one CUDA graph; "
                                                         "needs --device-resident")
    ap.add_argument("--dropout", type=int, default=None, metavar="SEED",
                    help="train with evaluation=False: the lifting stage's dropout, seeded with SEED")
    args = ap.parse_args()
    if args.graph and not args.device_resident:
        ap.error("--graph captures the reader too, which needs --device-resident")
    VARIANT = args.variant
    train_para.update(max_iter=args.iters, show_loss_freq=args.show_loss_freq, snapshot_freq=args.snapshot_freq or args.iters + 1,
                      snapshot_dir=args.snapshot_dir or train_para['snapshot_dir'] % VARIANT)

    path, tmp = db_path(args.db, "rhd", 16)
    try:
        # training_lifting.py:44-46 reads with shuffle=True and four noise flags; --augment does the same (seeded draws, not TF's
        # streams).  The default reads in file order without noise, as the losses recorded in DESIGN.md section 6 were measured.
        if args.augment:
            dataset = BinaryDbReader(mode='training', batch_size=8, shuffle=True, hand_crop=True, use_wrist_coord=False, coord_uv_noise=True,
                                     crop_center_noise=True, crop_offset_noise=True, crop_scale_noise=True, path_to_db=path, seed=args.seed,
                                     device_resident=args.device_resident)
        else:
            dataset = BinaryDbReader(mode='training', batch_size=8, shuffle=False, hand_crop=True, use_wrist_coord=False, path_to_db=path,
                                     device_resident=args.device_resident)

        net = PosePriorNetwork(VARIANT)
        ctx = runtime.default_context()
        ctx.set_precision('bf16x3')
        evaluation = args.dropout is None
        if not evaluation:
            ctx.set_dropout(args.dropout)
        # tf.global_variables_initializer() (:85)
        ctx.load_weights(Wt.xavier_weights(args.seed, bottleneck=VARIANT == 'bottleneck'))
        scopes = ['PosePrior', 'ViewpointNet'] if VARIANT == 'proposed' else ['PosePrior']
        variables = {}
        for scope in scopes:
            variables.update(ctx.variables(scope))

        # Solver (:79-83): minimize() over every trainable variable of the graph, both scopes in 'proposed'.  It is called without
        # global_step, so the reference's learning rate stays lr[0]; --advance-global-step makes the schedule take effect.
        lr_scheduler = LearningRateScheduler(values=train_para['lr'], steps=train_para['lr_iter'])
        global_step = 0
        opt = Adam(list(variables.values()), lr=lr_scheduler.get_lr(global_step))

        if not os.path.exists(train_para['snapshot_dir']):
            os.mkdir(train_para['snapshot_dir'])
            print('Created snapshot dir:', train_para['snapshot_dir'])

        def iteration():
            data = dataset.get()
            _, coord3d_pred, R = net.inference(data['scoremap'], data['hand_side'], evaluation, train=True)  # :53-54
            if VARIANT in ('direct', 'bottleneck'):                                                          # :62-76
                loss = A.mse_loss(coord3d_pred, data['keypoint_xyz21_normed'])
            elif VARIANT == 'local':
                loss = A.mse_loss(coord3d_pred, data['keypoint_xyz21_local'])
            elif VARIANT == 'local_w_xyz_loss':
                loss = A.mse_loss(bone_rel_trafo_inv(coord3d_pred), data['keypoint_xyz21_normed'])
            else:
                loss = A.mse_loss(coord3d_pred, data['keypoint_xyz21_can']) + A.mse_loss(R, data['rot_mat'])
            opt.zero_grad()
            loss.backward()
            opt.step()
            return loss.detach()

        run = GraphedIteration(iteration) if args.graph else iteration
        print('Starting to train ...')
        for i in range(train_para['max_iter']):
            opt.set_lr(lr_scheduler.get_lr(global_step))          # outside the iteration: a graph replays device work only
            loss = run()
            if args.advance_global_step:
                global_step += 1

            if (i % train_para['show_loss_freq']) == 0:
                print('Iteration %d\t Loss %.1e' % (i, float(loss.detach())))
                sys.stdout.flush()

            if (i % train_para['snapshot_freq']) == 0:
                Wt.save_weight_file('%s/model-%d.pickle' % (train_para['snapshot_dir'], i), variables)
                print('Saved a snapshot.')
                sys.stdout.flush()

        print('Training finished. Saving final snapshot.')
        Wt.save_weight_file('%s/model-%d.pickle' % (train_para['snapshot_dir'], train_para['max_iter']), variables)
    finally:
        cleanup(tmp)

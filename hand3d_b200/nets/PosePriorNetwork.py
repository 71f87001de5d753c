"""PosePriorNetwork -- lifting 2D score maps to 3D behind the reference's API
(nets/PosePriorNetwork.py:29-159).  All five variants ('direct', 'bottleneck', 'local',
'local_w_xyz_loss', 'proposed') run on the same sm_90a kernels as ColorHandPose3DNetwork; the 'local*' variants add
the forward-kinematics kernel that replaces bone_rel_trafo_inv (utils/relative_trafo.py:243-295).
"""
from __future__ import annotations

import os

import torch

from .. import autograd as A, runtime, weights as _weights


class PosePriorNetwork(object):
    """ Network containing different variants for lifting 2D predictions into 3D. """
    def __init__(self, variant):
        self.num_kp = 21
        self.variant = variant

    def init(self, session=None, weight_files=None, exclude_var_list=None, weights=None):
        """ Initializes weights from pickled python dictionaries (reference :36-57). """
        if exclude_var_list is None:
            exclude_var_list = list()
        ctx = runtime.default_context()
        if weights is not None:
            wd = {k: v for k, v in weights.items() if not any([x in k for x in exclude_var_list])}
            ctx.load_weights(wd)
            print('Loaded %d variables from %s' % (len(wd), 'memory'))
            return
        for file_name in weight_files:
            assert os.path.exists(file_name), "File not found."
            wd = _weights.load_weight_files([file_name], exclude_var_list, verbose=False)
            if len(wd) > 0:
                ctx.load_weights(wd)
                print('Loaded %d variables from %s' % (len(wd), file_name))

    def inference(self, scoremap, hand_side, evaluation=True, train=False):
        """ Infere 3D coordinates from 2D scoremaps (reference :59-95).

            scoremap [B,256,256,21] -> avg_pool 8x8 -> variant.  Returns (coord_xyz_rel_normed, coord3d, R).

            train=True builds the graph from hand3d_b200.autograd over ctx.variables('PosePrior') (and ctx.variables('ViewpointNet')
            for 'proposed'), as the reference's own inference() does with trainable variables (training_lifting.py:54): a loss of
            coord3d, R or coord_xyz_rel_normed back-propagates into those Parameters.  The 8x8 average pool takes no gradient.

            evaluation=False applies the dropout layers after fc_rel0 / fc_rel1 (keep 0.8) and fc_vp0 / fc_vp1 (keep 0.75, 'proposed'),
            drawn from the context's seeded generator (runtime.default_context().set_dropout(seed)); one call is one draw.
        """
        from .ColorHandPose3DNetwork import _dropout_wanted
        drop = _dropout_wanted(evaluation)
        ctx = runtime.default_context()
        scoremap_pooled = ctx.avg_pool8(scoremap)                       # :61
        if train:
            return self._train_inference(scoremap_pooled, hand_side, drop)
        if self.variant in ('direct', 'bottleneck'):
            c, _, _ = ctx.lifting(scoremap_pooled, hand_side, self.variant, dropout=drop)
            return c, c, None
        elif self.variant in ('local', 'local_w_xyz_loss'):
            # :70-75 -- the net predicts bone-relative coords; bone_rel_trafo_inv (utils/relative_trafo.py:243) assembles xyz
            normed, rel, _ = ctx.lifting(scoremap_pooled, hand_side, 'local', dropout=drop)
            return normed, rel, None
        elif self.variant == 'proposed':
            out, can, R = ctx.lifting(scoremap_pooled, hand_side, 'proposed', dropout=drop)
            return out, can, R
        else:
            assert 0, "Unknown variant."

    def _train_inference(self, scoremap_pooled, hand_side, drop=False):
        from .ColorHandPose3DNetwork import _train_advance, _train_pose3d_can, _train_rotate, _train_viewpoint_u
        if self.variant in ('direct', 'bottleneck'):
            c = _train_pose3d_can(scoremap_pooled, hand_side, bottleneck=self.variant == 'bottleneck', dropout=drop)
            r = c, c, None
        elif self.variant in ('local', 'local_w_xyz_loss'):
            rel = _train_pose3d_can(scoremap_pooled, hand_side, dropout=drop)
            r = A.bone_rel_trafo_inv(rel), rel, None
        elif self.variant == 'proposed':
            can = _train_pose3d_can(scoremap_pooled, hand_side, dropout=drop)
            R, out = _train_rotate(can, _train_viewpoint_u(scoremap_pooled, hand_side, dropout=drop), hand_side)
            r = out, can, R
        else:
            assert 0, "Unknown variant."
        _train_advance(drop)
        return r

"""ColorHandPose3DNetwork -- H100-native forward pass behind the reference's Python API
(nets/ColorHandPose3DNetwork.py:28-384): same class / method names, argument order, NHWC float32
tensors and return-tuple order, eager over torch CUDA tensors.  All arithmetic runs in
libhand3d_b200.so (hand-written sm_90a kernels); there is no TF session and no CPU fallback.
"""
from __future__ import annotations

import os

import torch

from .. import _lib, arch, autograd as A, runtime, weights as _weights


def _truthy(x):
    return bool(x.item()) if torch.is_tensor(x) else bool(x)


_TRAIN_PRECISIONS = {_lib.PRECISIONS["bf16x3"]: "bf16x3", _lib.PRECISIONS["bf16"]: "bf16"}


def _train_scope(scope):
    """(context, variables of scope, precision name) of a train=True graph; the convolution backward runs in bf16x3 or bf16 only."""
    ctx = runtime.default_context()
    prec = _TRAIN_PRECISIONS.get(ctx.precision)
    if prec is None:
        name = [k for k, v in _lib.PRECISIONS.items() if v == ctx.precision]
        raise ValueError("train=True needs the context precision 'bf16x3' or 'bf16' (the convolution backward runs in these two), "
                         "got %r" % (name[0] if name else ctx.precision))
    return ctx, ctx.variables(scope), prec


def _train_layers(x, v, scope, layers, pool_after, prec):
    """The conv_relu / max_pool chain of nets/ColorHandPose3DNetwork.py:150-157 (HandSegNet) and :189-199 (PoseNet2D)."""
    for name, k, stride, _, _, leaky in layers:
        x = A.conv2d(x, v["%s/%s/weights" % (scope, name)], v["%s/%s/biases" % (scope, name)], stride, leaky, prec)
        if name in pool_after:
            x = A.max_pool(x)
    return x


def _train_detection(image):
    ctx, v, prec = _train_scope("HandSegNet")
    image = image.to(torch.float32).contiguous()
    scoremap = _train_layers(image, v, "HandSegNet", arch.HANDSEGNET, arch.HANDSEGNET_POOL_AFTER, prec)
    return A.resize_bilinear(scoremap, image.shape[1], image.shape[2])       # :165-166


def _train_pose2d(image_crop, num_kp):
    ctx, v, prec = _train_scope("PoseNet2D")
    layers = {l[0]: l for l in arch.POSENET2D}
    trunk = [layers[n] for n in ("conv1_1", "conv1_2", "conv2_1", "conv2_2", "conv3_1", "conv3_2", "conv3_3", "conv3_4", "conv4_1",
                                 "conv4_2", "conv4_3", "conv4_4", "conv4_5", "conv4_6", "conv4_7")]
    encoding = _train_layers(image_crop.to(torch.float32).contiguous(), v, "PoseNet2D", trunk, arch.POSENET2D_POOL_AFTER, prec)
    scoremap_list = [_train_layers(encoding, v, "PoseNet2D", [layers["conv5_1"], layers["conv5_2"]], (), prec)]    # :202-204
    for pass_id in range(2):                                                                                      # :207-215
        x = torch.cat([scoremap_list[-1], encoding], 3)      # 21 + 128 = 149 channels: a plain copy, as tf.concat
        unit = [layers["conv%d_%d" % (pass_id + 6, i)] for i in range(1, 8)]
        scoremap_list.append(_train_layers(x, v, "PoseNet2D", unit, (), prec))
    assert all(s.shape[3] == num_kp for s in scoremap_list)
    return scoremap_list


def _dropout_wanted(evaluation):
    """True for evaluation=False: the lifting stage applies its dropout layers, which needs a seeded context (Context.set_dropout);
    without a seed evaluation=False raises NotImplementedError."""
    if _truthy(evaluation):
        return False
    runtime.default_context()._dropout_mode(True)
    return True


# the dropout layers of the lifting stage's FC stacks (nets/PosePriorNetwork.py:113-114, 151-154): (keep_prob, layer id) per hidden layer
_DROPOUT = {"fc_rel0": (_lib.DROPOUT_KEEP_POSEPRIOR, _lib.DROPOUT_LAYER_FC_REL0), "fc_rel1": (_lib.DROPOUT_KEEP_POSEPRIOR, _lib.DROPOUT_LAYER_FC_REL1),
            "fc_vp0": (_lib.DROPOUT_KEEP_VIEWPOINT, _lib.DROPOUT_LAYER_FC_VP0), "fc_vp1": (_lib.DROPOUT_KEEP_VIEWPOINT, _lib.DROPOUT_LAYER_FC_VP1)}


def _train_advance(dropout):
    """Ends one network forward: the next one draws new masks."""
    if dropout:
        runtime.default_context().dropout_advance()


def _train_lift_input(pooled, hand_side):
    return pooled.to(torch.float32).contiguous(), hand_side.to(torch.float32).contiguous()


def _train_fc_stack(x, hand_side, v, scope, names, prec, dropout=False):
    """Flatten (NHWC order, as tf.reshape), concat hand_side, then the leaky FC layers `names` (nets/PosePriorNetwork.py:110-114),
    each followed by its dropout layer when `dropout` (at the current draw; the caller advances it)."""
    x = torch.cat([x.reshape(x.shape[0], -1), hand_side], 1)
    for name in names:
        x = A.fully_connected(x, v["%s/%s/weights" % (scope, name)], v["%s/%s/biases" % (scope, name)], True, prec)
        if dropout:
            x = A.dropout(x, *_DROPOUT[name])
    return x


def _train_pose3d_can(pooled, hand_side, bottleneck=False, dropout=False):
    """PosePrior (nets/PosePriorNetwork.py:97-122) over ctx.variables('PosePrior'): [B,32,32,21], [B,2] -> [B,21,3].  dropout=True
    (evaluation=False) applies the dropout after fc_rel0 and fc_rel1 at the current draw."""
    _, v, prec = _train_scope("PosePrior")
    has_bn = "PosePrior/fc_bottleneck/weights" in v
    if bottleneck != has_bn:
        raise ValueError("the %s PosePrior needs %s fc_bottleneck layer in the loaded weights" % (
            "'bottleneck'" if bottleneck else "non-bottleneck", "an" if bottleneck else "no"))
    pooled, hand_side = _train_lift_input(pooled, hand_side)
    x = _train_layers(pooled, v, "PosePrior", arch.POSEPRIOR[:6], (), prec)
    x = _train_fc_stack(x, hand_side, v, "PosePrior", ("fc_rel0", "fc_rel1"), prec, dropout)
    if bottleneck:
        x = A.fully_connected(x, v["PosePrior/fc_bottleneck/weights"], v["PosePrior/fc_bottleneck/biases"], False, prec)
    x = A.fully_connected(x, v["PosePrior/fc_xyz/weights"], v["PosePrior/fc_xyz/biases"], False, prec)
    return x.view(x.shape[0], 21, 3)


def _train_viewpoint_u(pooled, hand_side, dropout=False):
    """ViewpointNet (nets/PosePriorNetwork.py:136-159) over ctx.variables('ViewpointNet') -> uxyz [B,3].  The three 128 -> 1 heads
    run as one 128 -> 3 layer whose weights are the concatenation of the three variables.  dropout=True applies the dropout after fc_vp0
    and fc_vp1 at the current draw."""
    _, v, prec = _train_scope("ViewpointNet")
    pooled, hand_side = _train_lift_input(pooled, hand_side)
    x = _train_layers(pooled, v, "ViewpointNet", arch.VIEWPOINT[:6], (), prec)
    x = _train_fc_stack(x, hand_side, v, "ViewpointNet", ("fc_vp0", "fc_vp1"), prec, dropout)
    heads = ["ViewpointNet/fc_vp_u%s" % a for a in "xyz"]
    w = torch.cat([v[h + "/weights"] for h in heads], 1)
    b = torch.cat([v[h + "/biases"] for h in heads], 0)
    return A.fully_connected(x, w, b, False, prec)


def _train_rotate(can, u, hand_side):
    """(R, out) of the 'proposed' lifting: Rodrigues, right-hand flip, out = flip(can) R."""
    return A.rotate_canonical(can, u, hand_side.to(torch.float32))


class ColorHandPose3DNetwork(object):
    """ Network performing 3D pose estimation of a human hand from a single color image. """
    def __init__(self):
        self.crop_size = 256
        self.num_kp = 21

    def init(self, session=None, weight_files=None, exclude_var_list=None, weights=None):
        """ Initializes weights from pickled python dictionaries (reference :34-59).

            session: ignored (kept for call-site compatibility; may be None)
            weight_files: list of str, pickle files {variable_name: ndarray}
            exclude_var_list: list of str, variables whose name contains any entry are not loaded
            weights: optional in-memory {variable_name: ndarray} (e.g. weights.synthetic_weights()) used
                     instead of files -- the released pickles cannot be downloaded offline.
        """
        if exclude_var_list is None:
            exclude_var_list = list()
        ctx = runtime.default_context()
        if weights is not None:
            wd = {k: v for k, v in weights.items() if not any([x in k for x in exclude_var_list])}
            ctx.load_weights(wd)
            print('Loaded %d variables from %s' % (len(wd), 'memory'))
            return
        if weight_files is None:
            weight_files = ['./weights/handsegnet-rhd.pickle', './weights/posenet3d-rhd-stb-slr-finetuned.pickle']
        for file_name in weight_files:
            assert os.path.exists(file_name), "File not found."
            wd = _weights.load_weight_files([file_name], exclude_var_list, verbose=False)
            if len(wd) > 0:
                ctx.load_weights(wd)     # unknown names raise ValueError, as assign_from_values does
                print('Loaded %d variables from %s' % (len(wd), file_name))

    def inference(self, image, hand_side, evaluation=True):
        """ Full pipeline: HandSegNet + PoseNet + PosePrior (reference :61-99).

            Returns (hand_scoremap [B,H,W,2], image_crop [B,256,256,3], scale_crop [B,1], center [B,2],
                     keypoints_scoremap [B,256,256,21], keypoint_coord3d [B,21,3]).

            evaluation=False applies the lifting stage's dropout (a seeded context: runtime.default_context().set_dropout(seed)).
        """
        r = runtime.default_context().pipeline(image, hand_side, with_pose3d=True, dropout=_dropout_wanted(evaluation))
        self.last_keypoints_uv = r["keypoints_uv"]
        return (r["hand_scoremap"], r["image_crop"], r["scale_crop"], r["center"], r["keypoints_scoremap"],
                r["keypoint_coord3d"])

    def inference2d(self, image):
        """ Only 2D part of the pipeline: HandSegNet + PoseNet (reference :101-129).

            Returns (keypoints_scoremap, image_crop, scale_crop, center) -- note the order differs from inference().
        """
        r = runtime.default_context().pipeline(image, None, with_pose3d=False)
        self.last_keypoints_uv = r["keypoints_uv"]
        return r["keypoints_scoremap"], r["image_crop"], r["scale_crop"], r["center"]

    @staticmethod
    def inference_detection(image, train=False):
        """ HandSegNet (reference :131-168): image [B,H,W,3] -> list of one [B,H,W,2] logits tensor.

            train=True builds the same graph from hand3d_b200.autograd over ctx.variables('HandSegNet'), so that a loss of its
            output back-propagates into those Parameters (training_handsegnet.py:47); H and W must be multiples of 8.
        """
        if train:
            return [_train_detection(image)]
        return [runtime.default_context().handsegnet(image)]

    def inference_pose2d(self, image_crop, train=False):
        """ PoseNet (reference :170-219): image_crop [B,256,256,3] -> list of three [B,32,32,21] score maps.

            train=True builds the same graph from hand3d_b200.autograd over ctx.variables('PoseNet2D') (training_posenet.py:47);
            the maps are then [B,H/8,W/8,21] for crops whose sides are multiples of 8.
        """
        if train:
            return _train_pose2d(image_crop, self.num_kp)
        return runtime.default_context().posenet(image_crop)

    def _inference_pose3d(self, keypoints_scoremap, hand_side, evaluation=True, train=False):
        """ PosePrior + Viewpoint (reference :221-247): [B,32,32,21], [B,2] -> [B,21,3].

            train=True builds the graph from hand3d_b200.autograd over ctx.variables('PosePrior') and ctx.variables('ViewpointNet').
            evaluation=False applies the dropout layers (a seeded context: runtime.default_context().set_dropout(seed)); one call is one
            draw.
        """
        drop = _dropout_wanted(evaluation)
        if train:
            can = _train_pose3d_can(keypoints_scoremap, hand_side, dropout=drop)
            out = _train_rotate(can, _train_viewpoint_u(keypoints_scoremap, hand_side, dropout=drop), hand_side)[1]
            _train_advance(drop)
            return out
        return runtime.default_context().lifting(keypoints_scoremap, hand_side, "proposed", dropout=drop)[0]

    @staticmethod
    def _optional_dropout(evaluation):
        # these two entries ignored `evaluation` before dropout existed: without a seed it stays the identity
        return not _truthy(evaluation) and runtime.default_context().dropout_seed is not None

    def _inference_pose3d_can(self, keypoints_scoremap, hand_side, evaluation=True, train=False):
        """ Canonical coordinates (reference :249-272).  evaluation=False on a seeded context applies PosePrior's dropout. """
        if train:
            drop = _dropout_wanted(evaluation)
            can = _train_pose3d_can(keypoints_scoremap, hand_side, dropout=drop)
            _train_advance(drop)
            return can
        return runtime.default_context().lifting(keypoints_scoremap, hand_side, "proposed", dropout=self._optional_dropout(evaluation))[1]

    def _inference_viewpoint(self, keypoints_scoremap, hand_side, evaluation=True, train=False):
        """ Viewpoint rotation matrix (reference :274-283).  evaluation=False on a seeded context applies ViewpointNet's dropout. """
        if train:
            drop = _dropout_wanted(evaluation)
            u = _train_viewpoint_u(keypoints_scoremap, hand_side, dropout=drop)
            _train_advance(drop)
            zeros = torch.zeros((u.shape[0], 21, 3), dtype=torch.float32, device=u.device)
            return _train_rotate(zeros, u, hand_side)[0]
        return runtime.default_context().lifting(keypoints_scoremap, hand_side, "proposed", dropout=self._optional_dropout(evaluation))[2]

    def _get_rot_mat(self, ux_b, uy_b, uz_b):
        """ Rodrigues rotation matrix from axis * angle (reference :311-334): three [B,1] -> [B,3,3]. """
        uxyz = torch.cat([ux_b, uy_b, uz_b], 1).contiguous()
        B = uxyz.shape[0]
        zeros = torch.zeros((B, 21, 3), dtype=torch.float32, device=uxyz.device)
        hs = torch.zeros((B, 2), dtype=torch.float32, device=uxyz.device); hs[:, 0] = 1
        return runtime.default_context().rotate_canonical(zeros, uxyz, hs)[0]

    @staticmethod
    def _flip_right_hand(coords_xyz_canonical, cond_right):
        """ Mirrors z where cond_right is true (reference :336-361). """
        B = coords_xyz_canonical.shape[0]
        cond = cond_right.reshape(B, -1)[:, 0] if torch.is_tensor(cond_right) else torch.as_tensor(cond_right).reshape(B, -1)[:, 0]
        return runtime.default_context().flip_right_hand(coords_xyz_canonical, cond.to(coords_xyz_canonical.device))

"""ColorHandPose3DNetwork -- H100-native forward pass behind the reference's Python API
(nets/ColorHandPose3DNetwork.py:28-384): same class / method names, argument order, NHWC float32
tensors and return-tuple order, eager over torch CUDA tensors.  All arithmetic runs in
libhand3d_b200.so (hand-written sm_90a kernels); there is no TF session and no CPU fallback.
"""
from __future__ import annotations

import os

import torch

from .. import runtime, weights as _weights


def _truthy(x):
    return bool(x.item()) if torch.is_tensor(x) else bool(x)


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
        """
        if not _truthy(evaluation):
            raise NotImplementedError("forward pass only: evaluation must be True (dropout is the identity)")
        r = runtime.default_context().pipeline(image, hand_side, with_pose3d=True)
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
        """ HandSegNet (reference :131-168): image [B,H,W,3] -> list of one [B,H,W,2] logits tensor. """
        if train:
            raise NotImplementedError("forward pass only: train must be False")
        return [runtime.default_context().handsegnet(image)]

    def inference_pose2d(self, image_crop, train=False):
        """ PoseNet (reference :170-219): image_crop [B,256,256,3] -> list of three [B,32,32,21] score maps. """
        if train:
            raise NotImplementedError("forward pass only: train must be False")
        return runtime.default_context().posenet(image_crop)

    def _inference_pose3d(self, keypoints_scoremap, hand_side, evaluation=True, train=False):
        """ PosePrior + Viewpoint (reference :221-247): [B,32,32,21], [B,2] -> [B,21,3]. """
        if not _truthy(evaluation) or train:
            raise NotImplementedError("forward pass only")
        return runtime.default_context().lifting(keypoints_scoremap, hand_side, "proposed")[0]

    def _inference_pose3d_can(self, keypoints_scoremap, hand_side, evaluation=True, train=False):
        """ Canonical coordinates (reference :249-272). """
        return runtime.default_context().lifting(keypoints_scoremap, hand_side, "proposed")[1]

    def _inference_viewpoint(self, keypoints_scoremap, hand_side, evaluation=True, train=False):
        """ Viewpoint rotation matrix (reference :274-283). """
        return runtime.default_context().lifting(keypoints_scoremap, hand_side, "proposed")[2]

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

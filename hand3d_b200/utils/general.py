"""H100-native mirror of the reference's utils/general.py hot-path helpers (same names, argument
order, NHWC layouts and return conventions), eager over torch CUDA tensors and backed by the
hand-written sm_90a kernels behind the C ABI (include/hand3d_b200.h).

Reference: utils/general.py:26-65,113-148 (NetworkOps), :163 crop_image_from_xy, :199 find_max_location,
:233 single_obj_scoremap, :271 calc_center_bb, :331 detect_keypoints, :347 trafo_coords.
EvalUtil (:522-611) is mirrored with a batched device path (SURVEY.md 8(f) row 3).
LearningRateScheduler (:480-519) is mirrored as a host function of an integer step.
Not mirrored (dead code in every graph / out of scope, SURVEY.md section 2): upconv*, spatial_dropout,
plot helpers, load_weights_from_snapshot.
"""
from __future__ import annotations

import contextlib

import numpy as np
import torch

from .. import runtime

_scope_stack = []


@contextlib.contextmanager
def variable_scope(name):
    """Stand-in for tf.variable_scope: NetworkOps looks variables up as '<scope>/<layer>/weights'."""
    _scope_stack.append(name)
    try:
        yield
    finally:
        _scope_stack.pop()


def _var(layer_name, what):
    scope = "/".join(_scope_stack)
    name = (scope + "/" if scope else "") + layer_name + "/" + what
    return runtime.default_context().dev_weight(name)


class NetworkOps(object):
    """Operations that are frequently used within networks (utils/general.py:26-160)."""
    neg_slope_of_relu = 0.01

    @classmethod
    def leaky_relu(cls, tensor, name='relu'):
        return runtime.default_context().leaky_relu(tensor)

    @classmethod
    def conv(cls, in_tensor, layer_name, kernel_size, stride, out_chan, trainable=True):
        w, b = _var(layer_name, "weights"), _var(layer_name, "biases")
        assert tuple(w.shape) == (kernel_size, kernel_size, in_tensor.shape[3], out_chan), "kernel shape mismatch for %s" % layer_name
        return runtime.default_context().conv2d(in_tensor, w, b, stride=stride, leaky=False)

    @classmethod
    def conv_relu(cls, in_tensor, layer_name, kernel_size, stride, out_chan, trainable=True):
        w, b = _var(layer_name, "weights"), _var(layer_name, "biases")
        assert tuple(w.shape) == (kernel_size, kernel_size, in_tensor.shape[3], out_chan), "kernel shape mismatch for %s" % layer_name
        return runtime.default_context().conv2d(in_tensor, w, b, stride=stride, leaky=True)

    @classmethod
    def max_pool(cls, bottom, name='pool'):
        return runtime.default_context().max_pool(bottom)

    @staticmethod
    def fully_connected(in_tensor, layer_name, out_chan, trainable=True):
        assert in_tensor.dim() == 2, 'Input to a fully connected layer must be a vector.'
        w, b = _var(layer_name, "weights"), _var(layer_name, "biases")
        assert tuple(w.shape) == (in_tensor.shape[1], out_chan)
        return runtime.default_context().fully_connected(in_tensor, w, b, leaky=False)

    @classmethod
    def fully_connected_relu(cls, in_tensor, layer_name, out_chan, trainable=True):
        assert in_tensor.dim() == 2, 'Input to a fully connected layer must be a vector.'
        w, b = _var(layer_name, "weights"), _var(layer_name, "biases")
        assert tuple(w.shape) == (in_tensor.shape[1], out_chan)
        return runtime.default_context().fully_connected(in_tensor, w, b, leaky=True)

    @staticmethod
    def dropout(in_tensor, keep_prob, evaluation):
        """Identity at evaluation time (utils/general.py:139-148); training is out of scope."""
        if not bool(evaluation):
            raise NotImplementedError("hand3d_b200 implements the forward pass only (evaluation must be True)")
        return in_tensor


def crop_image_from_xy(image, crop_location, crop_size, scale=1.0):
    """utils/general.py:163-196.  image [B,H,W,C], crop_location [B,2] (row, col), scale [B,1] / scalar."""
    assert image.dim() == 4, "Image needs to be of shape [batch, width, height, channel]"
    B = image.shape[0]
    if not torch.is_tensor(scale):
        scale = torch.full((B,), float(scale), dtype=torch.float32, device=image.device)
    crop_location = torch.as_tensor(crop_location, device=image.device)
    return runtime.default_context().crop_image_from_xy(image.to(torch.float32), crop_location, int(crop_size), scale)


def _seg(scoremap):
    assert scoremap.dim() == 4, "Scoremap must be 4D."
    return runtime.default_context().seg_postprocess(scoremap)


def find_max_location(scoremap):
    """utils/general.py:199-230: first-occurrence arg-max per image -> [B,2] int32 (row, col).

    Accepts [B,H,W], [B,H,W,1] or [H,W] fg score maps.  (The kernel arg-maxes any fp32 map: it is fed
    through the 2-class seg kernel as logits (0, x) only when a probability map is not available, so here
    a dedicated path is used.)"""
    s = scoremap
    if s.dim() == 4:
        s = s.squeeze(3)
    if s.dim() == 2:
        s = s.unsqueeze(0)
    assert s.dim() == 3, "Scoremap must be 3D."
    uv = runtime.default_context().detect_keypoints(s.unsqueeze(3).contiguous())   # [B,1,2]
    return uv[:, 0, :]


def single_obj_scoremap(scoremap):
    """utils/general.py:233-268: [B,H,W,2] logits -> [B,H,W,1] float32 {0,1} object mask."""
    return _seg(scoremap)["hand_mask"].to(torch.float32).unsqueeze(3)


def calc_center_bb(binary_class_mask):
    """utils/general.py:271-328: mask [B,H,W,1] / [B,H,W] -> (center [B,2], bb [B,2,2], crop_size [B,1]); one kernel
    (h3d_calc_center_bb): bounding box of the pixels with int(mask) == 1, the reference's fall-backs for an empty mask."""
    m = binary_class_mask
    if m.dim() == 4:
        m = m.squeeze(3)
    assert m.dim() == 3, "binary_class_mask must be 3D."
    return runtime.default_context().calc_center_bb(m.to(torch.float32).contiguous())


def detect_keypoints(scoremaps):
    """utils/general.py:331-344.  numpy [H,W,C] / [1,H,W,C] -> float64 [C,2] (v,u) like the reference;
    a torch CUDA tensor [B,H,W,C] / [H,W,C] -> int32 [B,C,2] / [C,2] on device."""
    if isinstance(scoremaps, np.ndarray):
        if len(scoremaps.shape) == 4:
            scoremaps = np.squeeze(scoremaps)
        s = scoremaps.shape
        assert len(s) == 3, "This function was only designed for 3D Scoremaps."
        assert (s[2] < s[1]) and (s[2] < s[0]), "Probably the input is not correct, because [H, W, C] is expected."
        ctx = runtime.default_context()
        t = torch.from_numpy(np.ascontiguousarray(scoremaps, np.float32)).to(ctx.device).unsqueeze(0)
        return ctx.detect_keypoints(t)[0].cpu().numpy().astype(np.float64)
    s = scoremaps
    squeeze = s.dim() == 3
    if squeeze:
        s = s.unsqueeze(0)
    uv = runtime.default_context().detect_keypoints(s)
    return uv[0] if squeeze else uv


def trafo_coords(keypoints_crop_coords, centers, scale, crop_size):
    """utils/general.py:347-357: (kp - crop_size//2) / scale + centers (numpy or torch, batched or not)."""
    if isinstance(keypoints_crop_coords, np.ndarray):
        keypoints_coords = np.copy(keypoints_crop_coords)
        keypoints_coords -= crop_size // 2
        keypoints_coords /= scale
        keypoints_coords += centers
        return keypoints_coords
    k = keypoints_crop_coords.to(torch.float64) - (crop_size // 2)
    scale = torch.as_tensor(scale, device=k.device, dtype=torch.float64)
    centers = torch.as_tensor(centers, device=k.device, dtype=torch.float64)
    if k.dim() == 3:
        scale = scale.reshape(-1, 1, 1)
        centers = centers.reshape(-1, 1, 2)
    return k / scale + centers


class LearningRateScheduler:
    """ Multistep learning-rate schedule (utils/general.py:480-519) evaluated on the host for an integer step.

        get_lr(step) returns the value TF's graph yields, as a float32, with the reference's branch quirks:
        one value: constant; two values: values[1] where step > steps[0] (strict), else values[0];
        n > 2 values: the sum of the values whose condition holds, the conditions being step < steps[0],
        steps[i] <= step < steps[i+1] and step >= steps[-1].
    """
    def __init__(self, steps, values):
        self.steps = steps
        self.values = values

        assert len(steps)+1 == len(values), "There must be one more element in value as step."

    def get_lr(self, global_step):
        step = int(global_step)
        vals = [np.float32(v) for v in self.values]
        if len(vals) == 1:
            return vals[0]
        if len(vals) == 2:
            return vals[1] if step > self.steps[0] else vals[0]
        conds = [step < self.steps[0]]
        conds += [self.steps[i] <= step < self.steps[i + 1] for i in range(len(self.steps) - 1)]
        conds.append(step >= self.steps[-1])
        return np.sum(np.where(conds, np.array(vals, np.float32), np.float32(0)), dtype=np.float32)


class EvalUtil:
    """ Util class for evaluation networks (utils/general.py:522-611): end-point error, PCK curve and AUC per key-point.

        feed() keeps the reference's single-sample numpy semantics and additionally accepts batches of torch CUDA
        tensors ([B,K,D] ground truth / prediction, [B,K] visibility): distances are then computed on the device by one
        kernel and only B*K floats travel to the host.  get_measures() returns the same 5-tuple as the reference.
    """
    def __init__(self, num_kp=21):
        self.num_kp = num_kp
        self.data = [list() for _ in range(num_kp)]

    def feed(self, keypoint_gt, keypoint_vis, keypoint_pred):
        if torch.is_tensor(keypoint_gt) and keypoint_gt.is_cuda:
            gt = keypoint_gt.to(torch.float32).reshape(-1, self.num_kp, keypoint_gt.shape[-1]).contiguous()
            pred = torch.as_tensor(keypoint_pred, device=gt.device).to(torch.float32).reshape(gt.shape).contiguous()
            vis = torch.as_tensor(keypoint_vis, device=gt.device).reshape(gt.shape[0], self.num_kp)
            dist = runtime.default_context().eval_keypoint_dist(gt, vis != 0, pred).cpu().numpy()
            for i in range(self.num_kp):
                col = dist[:, i]
                self.data[i].extend(col[col >= 0].tolist())
            return
        keypoint_gt = np.squeeze(np.asarray(keypoint_gt))
        keypoint_pred = np.squeeze(np.asarray(keypoint_pred))
        keypoint_vis = np.squeeze(np.asarray(keypoint_vis)).astype('bool')
        assert len(keypoint_gt.shape) == 2
        assert len(keypoint_pred.shape) == 2
        assert len(keypoint_vis.shape) == 1
        euclidean_dist = np.sqrt(np.sum(np.square(keypoint_gt - keypoint_pred), axis=1))
        for i in range(keypoint_gt.shape[0]):
            if keypoint_vis[i]:
                self.data[i].append(euclidean_dist[i])

    def _get_pck(self, kp_id, threshold):
        if len(self.data[kp_id]) == 0:
            return None
        return np.mean((np.array(self.data[kp_id]) <= threshold).astype('float'))

    def _get_epe(self, kp_id):
        if len(self.data[kp_id]) == 0:
            return None, None
        d = np.array(self.data[kp_id])
        return np.mean(d), np.median(d)

    def get_measures(self, val_min, val_max, steps):
        """ (mean EPE, median EPE, AUC, PCK curve, thresholds), each averaged over the key-points that have data. """
        trapz = getattr(np, "trapezoid", None) or np.trapz
        thresholds = np.linspace(val_min, val_max, steps)
        norm_factor = trapz(np.ones_like(thresholds), thresholds)
        means, medians, aucs, curves = [], [], [], []
        for part_id in range(self.num_kp):
            mean, median = self._get_epe(part_id)
            if mean is None:
                continue                      # no valid measurement for this key-point
            means.append(mean)
            medians.append(median)
            curve = np.array([self._get_pck(part_id, t) for t in thresholds])
            curves.append(curve)
            aucs.append(trapz(curve, thresholds) / norm_factor)
        return (np.mean(np.array(means)), np.mean(np.array(medians)), np.mean(np.array(aucs)), np.mean(np.array(curves), 0),
                thresholds)

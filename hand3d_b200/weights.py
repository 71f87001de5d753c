"""Weight dictionaries in the reference's pickle layout (SURVEY.md 8a.2).

* ``load_weight_files`` mirrors ColorHandPose3DNetwork.init (nets/ColorHandPose3DNetwork.py:34-59):
  pickled ``{variable_name: ndarray}``; names containing any ``exclude_var_list`` substring are dropped.
* ``synthetic_weights`` generates seeded random-init weights with exactly the reference's variable
  names and shapes (the released pickles are not available offline).
"""
from __future__ import annotations

import os
import pickle

import numpy as np

from . import arch

# HandSegNet/conv6_2 bias shift for class 1 ("hand"): keeps the synthetic foreground fraction in
# the 10-40 % range so that masks / bounding boxes are non-degenerate (SURVEY.md 8d).
# Calibrated on the oracle: +0.85 gives ~10 % foreground on the seed-1 noise images; +0.15 gives
# small corner masks on ``synthetic_blob_images`` (crops that leave the image -> extrapolation).
SEG_FG_LOGIT_SHIFT = 0.85


def synthetic_weights(seed: int = 0, bottleneck: bool = False, dtype=np.float32, seg_shift: float = SEG_FG_LOGIT_SHIFT):
    """He-init for leaky-ReLU(0.01): W ~ N(0, 2/((1+0.01^2) fan_in)), b ~ N(0, 0.01^2)."""
    rng = np.random.default_rng(seed)
    out = {}
    for name, shape in arch.variable_shapes(bottleneck).items():
        if name.endswith("/weights"):
            fan_in = int(np.prod(shape[:-1]))
            std = np.sqrt(2.0 / ((1.0 + 0.01 ** 2) * fan_in))
            out[name] = (rng.standard_normal(shape) * std).astype(dtype)
        else:
            out[name] = (rng.standard_normal(shape) * 0.01).astype(dtype)
    out["HandSegNet/conv6_2/biases"] = out["HandSegNet/conv6_2/biases"] + np.array(
        [0.0, seg_shift], dtype)
    return out


def load_weight_files(weight_files, exclude_var_list=None, verbose=True):
    """nets/ColorHandPose3DNetwork.py:42-59 (same asserts / messages, no TF session)."""
    if exclude_var_list is None:
        exclude_var_list = list()
    merged = {}
    for file_name in weight_files:
        assert os.path.exists(file_name), "File not found."
        with open(file_name, "rb") as fi:
            try:
                weight_dict = pickle.load(fi)
            except UnicodeDecodeError:  # python-2 pickles
                fi.seek(0)
                weight_dict = pickle.load(fi, encoding="latin1")
        weight_dict = {k: v for k, v in weight_dict.items() if not any([x in k for x in exclude_var_list])}
        if len(weight_dict) > 0:
            merged.update({k: np.asarray(v, np.float32) for k, v in weight_dict.items()})
            if verbose:
                print("Loaded %d variables from %s" % (len(weight_dict), file_name))
    return merged


def save_weight_file(path, variables):
    """Writes a snapshot in the reference's pickle layout ({variable_name: float32 ndarray}, pickle protocol 2), which
    ColorHandPose3DNetwork().init(weight_files=[path]) loads back.  variables: {name: ndarray or tensor}, e.g. ctx.variables(scope)."""
    out = {}
    for name, v in variables.items():
        if hasattr(v, "detach"):
            v = v.detach().cpu().numpy()
        out[name] = np.ascontiguousarray(v, dtype=np.float32)
    tmp = path + ".tmp"
    with open(tmp, "wb") as f:
        pickle.dump(out, f, protocol=2)
    os.replace(tmp, path)
    return path


def validate(weight_dict, known=None):
    """Unknown names raise (as tf.contrib.framework.assign_from_values does); shapes must match."""
    known = known or {**arch.variable_shapes(False), **arch.variable_shapes(True)}
    for k, v in weight_dict.items():
        if k not in known:
            raise ValueError("Unknown variable name: %s" % k)
        exp = known[k]
        if k == "PosePrior/fc_xyz/weights" and tuple(v.shape) in ((512, 63), (30, 63)):
            continue
        if tuple(v.shape) != tuple(exp):
            raise ValueError("Shape mismatch for %s: %s vs %s" % (k, tuple(v.shape), tuple(exp)))


def synthetic_images(batch: int, H: int = 320, W: int = 320, seed: int = 1):
    """uint8 ~ U{0..255} -> x/255 - 0.5 (reference preprocessing run.py:59)."""
    rng = np.random.default_rng(seed)
    u8 = rng.integers(0, 256, size=(batch, H, W, 3), dtype=np.uint8)
    return (u8.astype(np.float32) / np.float32(255.0) - np.float32(0.5)).astype(np.float32)


def synthetic_blob_images(batch: int, H: int = 320, W: int = 320, seed: int = 1):
    """Soft ellipses composited over low-amplitude noise: spatially structured inputs that give the
    segmentation branch diverse masks (SURVEY.md 8d "mask-diversity tests")."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    out = np.empty((batch, H, W, 3), np.float32)
    for b in range(batch):
        img = rng.normal(0.0, 0.08, size=(H, W, 3)).astype(np.float32)
        for _ in range(int(rng.integers(1, 4))):
            cy, cx = rng.uniform(0.15, 0.85) * H, rng.uniform(0.15, 0.85) * W
            ry, rx = rng.uniform(0.06, 0.25) * H, rng.uniform(0.06, 0.25) * W
            col = rng.uniform(-0.5, 0.5, size=3).astype(np.float32)
            d = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2
            a = (1.0 / (1.0 + np.exp(np.minimum((d - 1.0) * 6.0, 60.0)))).astype(np.float32)[..., None]
            img = img * (1 - a) + col * a
        out[b] = np.clip(img, -0.5, 0.5)
    return out


def synthetic_hand_side(batch: int, seed: int = 2):
    rng = np.random.default_rng(seed)
    right = rng.integers(0, 2, size=batch)
    hs = np.zeros((batch, 2), np.float32)
    hs[np.arange(batch), right] = 1.0
    return hs

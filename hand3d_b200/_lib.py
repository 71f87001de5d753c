"""ctypes binding of libhand3d_b200.so (include/hand3d_b200.h).

There is deliberately no fallback: if the shared library is missing and cannot be built, or a compute
entry point fails (e.g. no sm_90a device), a RuntimeError is raised with h3d_last_error().
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libhand3d_b200.so")

OK, EINVAL, ENODEVICE, ECUDA, EWEIGHTS, EWORKSPACE = 0, -1, -2, -3, -4, -5
PREC_FP32_FFMA, PREC_BF16X3, PREC_FP16X3, PREC_FP16, PREC_BF16 = 0, 1, 2, 3, 4
PRECISIONS = {"fp32_ffma": 0, "bf16x3": 1, "fp16x3": 2, "fp16": 3, "bf16": 4, "fp16_f8c": 5}
VARIANTS = {"direct": 0, "bottleneck": 1, "proposed": 2, "local": 3, "local_w_xyz_loss": 3}

_p, _i, _i64, _f = C.c_void_p, C.c_int, C.c_int64, C.c_float

# name -> (restype, argtypes); mirrors include/hand3d_b200.h one to one
SIGNATURES = {
    "h3d_last_error": (C.c_char_p, []),
    "h3d_version": (_i, []),
    "h3d_device_available": (_i, []),
    "h3d_create": (_i, [C.POINTER(_p), _i]),
    "h3d_destroy": (_i, [_p]),
    "h3d_set_precision": (_i, [_p, _i]),
    "h3d_get_precision": (_i, [_p]),
    "h3d_set_tuning": (_i, [_p, C.c_char_p, _i]),
    "h3d_check_errors": (_i, [_p, C.POINTER(_i)]),
    "h3d_launch_count": (_i64, [_p]),
    "h3d_profile_begin": (_i, [_p]),
    "h3d_profile_end": (_i, [_p, C.POINTER(C.c_double), C.POINTER(_i64), C.POINTER(_i64)]),
    "h3d_load_weight": (_i, [_p, C.c_char_p, _p, C.POINTER(_i64), _i]),
    "h3d_scope_ready": (_i, [_p, C.c_char_p]),
    "h3d_workspace_bytes": (_i64, [_p, _i, _i, _i]),
    "h3d_set_workspace": (_i, [_p, _p, _i64]),
    "h3d_handsegnet_forward": (_i, [_p, _p, _i, _i, _i, _p, _p]),
    "h3d_posenet_forward": (_i, [_p, _p, _i, _i, _i, _p, _p, _p, _p]),
    "h3d_lifting_forward": (_i, [_p, _p, _p, _i, _i, _p, _p, _p, _p]),
    "h3d_pipeline_forward": (_i, [_p, _p, _p, _i, _i, _i, _i, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "h3d_pose2d_forward": (_i, [_p, _p, _i, _i, _i, _p, _p, _p]),
    "h3d_conv2d_f32": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _p]),
    "h3d_conv2d_tc": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _p]),
    "h3d_conv2d_tc_strided": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p]),
    "h3d_pack_conv_weights": (_i, [_p, _p, _p, _i, _i, _i, _i, C.POINTER(_p)]),
    "h3d_free_packed_conv": (_i, [_p, _p]),
    "h3d_conv2d_tc_packed": (_i, [_p, _p, _p, _p, _i, _i, _i, _i, _i, _p]),
    "h3d_conv2d_tc_dev": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p]),
    "h3d_conv2d_tc_backward": (_i, [_p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p]),
    "h3d_leaky_relu_f32": (_i, [_p, _p, _p, _i64, _p]),
    "h3d_maxpool2x2_f32": (_i, [_p, _p, _p, _i, _i, _i, _i, _p]),
    "h3d_maxpool2x2_backward_f32": (_i, [_p, _p, _p, _p, _i, _i, _i, _i, _p]),
    "h3d_fully_connected_f32": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _i, _p]),
    "h3d_resize_bilinear_tf1": (_i, [_p, _p, _p, _i, _i, _i, _i, _i, _i, _p]),
    "h3d_avgpool8": (_i, [_p, _p, _p, _i, _i, _i, _i, _p]),
    "h3d_seg_postprocess": (_i, [_p, _p, _i, _i, _i, _p, _p, _p, _p, _p, _p]),
    "h3d_calc_center_bb": (_i, [_p, _p, _i, _i, _i, _p, _p, _p, _p]),
    "h3d_crop_image_from_xy": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _p]),
    "h3d_detect_keypoints": (_i, [_p, _p, _i, _i, _i, _i, _p, _p]),
    "h3d_upsample_detect_keypoints": (_i, [_p, _p, _i, _i, _i, _i, _i, _p, _p, _p]),
    "h3d_pack_records": (_i, [_p, _p, _p, _p, _p, _i, _p, _p]),
    "h3d_gather_records_p2p": (_i, [_p, _p, _p, _p, _p, _i, _i, _p, _p, C.c_uint64, _i, _i, C.c_uint32, _i64, _p]),
    "h3d_decode_records": (_i, [_p, _i, _p, _i, _i, _p, _p, _p, _p, _p]),
    "h3d_rhd_reader_items": (_i, [_p, _p, _p, _p, _i, _i, _i, _i, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "h3d_stb_reader_items": (_i, [_p, _p, _i, _i, _p, _p, _p, _p, _p, _p]),
    "h3d_gaussian_scoremap": (_i, [_p, _p, _p, _i, _i, _i, _i, _f, _p, _p]),
    "h3d_canonical_trafo": (_i, [_p, _p, _p, _i, _p, _p, _p, _p]),
    "h3d_eval_keypoint_dist": (_i, [_p, _p, _p, _p, _i, _i, _p, _p]),
    "h3d_bone_rel_trafo_inv": (_i, [_p, _p, _p, _i, _p]),
    "h3d_rotate_canonical": (_i, [_p, _p, _p, _p, _i, _p, _p, _p]),
    "h3d_flip_right_hand": (_i, [_p, _p, _p, _i, _p, _p]),
    "h3d_resize_bilinear_tf1_backward": (_i, [_p, _p, _p, _i, _i, _i, _i, _i, _i, _p]),
    "h3d_scoremap_loss_forward": (_i, [_p, _p, _p, _p, _i, _i, _i, _p, _p, _p]),
    "h3d_scoremap_loss_backward": (_i, [_p, _p, _p, _p, _p, _p, _i, _i, _i, _p, _p]),
    "h3d_softmax_xent_forward": (_i, [_p, _p, _p, _i64, _p, _p]),
    "h3d_softmax_xent_backward": (_i, [_p, _p, _p, _p, _i64, _p, _p]),
    "h3d_adam_state_set": (_i, [_p, _p, _f, _f, _f, _p]),
    "h3d_adam_set_lr": (_i, [_p, _p, _f, _p]),
    "h3d_adam_step": (_i, [_p, _p, _i, _p, _f, _f, _f, _p]),
}
ADAM_STATE_WORDS = 4   # H3D_ADAM_STATE_WORDS

_lib = None


def load():
    """Loads (building in-tree with nvcc if necessary) the shared library; raises if impossible."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        from . import build as _build
        _build.build()
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)   # AttributeError if the header and the library drifted apart
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error() -> str:
    return load().h3d_last_error().decode("utf-8", "replace")


def check(rc: int, what: str = ""):
    if rc != OK:
        raise RuntimeError("hand3d_b200: %s failed (code %d): %s" % (what or "call", rc, last_error()))

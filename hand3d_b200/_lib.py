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
# kernels of the CUDA-core convolution (H3D_DIRECT_*) and the split-K scratch the entries give it (H3D_CONV_SPLITK_SCRATCH_FLOATS)
DIRECT_KERNELS = {0: "c3_tc", 1: "c3_ffma", 2: "vec", 3: "scalar"}
CONV_SPLITK_SCRATCH_FLOATS = 600 * 64 * 64
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
    "h3d_fill_scratch": (_i, [_p, _i, _p]),
    "h3d_handsegnet_forward": (_i, [_p, _p, _i, _i, _i, _p, _p]),
    "h3d_posenet_forward": (_i, [_p, _p, _i, _i, _i, _p, _p, _p, _p]),
    "h3d_lifting_forward": (_i, [_p, _p, _p, _i, _i, _p, _p, _p, _p]),
    "h3d_pipeline_forward": (_i, [_p, _p, _p, _i, _i, _i, _i, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "h3d_pose2d_forward": (_i, [_p, _p, _i, _i, _i, _p, _p, _p]),
    "h3d_track_state_bytes": (_i64, [_i]),
    "h3d_track_step": (_i, [_p, _p, _p, _i, _i, _i, _i, _i, _f, _f, _p, _p, _p, _p, _p, _p, _p, _p]),
    "h3d_track_update": (_i, [_p, _p, _p, _p, _p, _i, _f, _f, _p, _p]),
    "h3d_track_step_slots": (_i, [_p, _p, _p, _i, _i, _i, _i, _f, _f, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "h3d_conv2d_f32": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _p]),
    "h3d_conv2d_tc": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _p]),
    "h3d_conv2d_tc_strided": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p]),
    "h3d_pack_conv_weights": (_i, [_p, _p, _p, _i, _i, _i, _i, C.POINTER(_p)]),
    "h3d_free_packed_conv": (_i, [_p, _p]),
    "h3d_conv2d_tc_packed": (_i, [_p, _p, _p, _p, _i, _i, _i, _i, _i, _p]),
    "h3d_conv2d_tc_dev": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p]),
    "h3d_conv2d_tc_backward": (_i, [_p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _i, _p]),
    "h3d_conv2d_layer_planes": (_i, [_p, _p, _i, _i, _i, _i, _p, _p, _i, _i, _i, _p, _i, _i, _i, _i, _p, _p, _p, _p, _i, _i, _p, _i, _i, _p]),
    "h3d_conv2d_tc_geometry": (_i, [_i, _i, _i, _i, _i, _i, C.POINTER(_i)]),
    "h3d_conv2d_wgrad_geometry": (_i, [_i, _i, _i, _i, _i, _i, C.POINTER(_i)]),
    "h3d_conv2d_f32_geometry": (_i, [_i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i64, C.POINTER(_i)]),
    "h3d_leaky_relu_f32": (_i, [_p, _p, _p, _i64, _p]),
    "h3d_maxpool2x2_f32": (_i, [_p, _p, _p, _i, _i, _i, _i, _p]),
    "h3d_maxpool2x2_backward_f32": (_i, [_p, _p, _p, _p, _i, _i, _i, _i, _p]),
    "h3d_fully_connected_f32": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _i, _p]),
    "h3d_fully_connected_f32_geometry": (_i, [_i, _i, _i, C.POINTER(_i)]),
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
    "h3d_reader_aug_params": (_i, [_p, _p, _i, C.c_uint64, _i, _p, _p]),
    "h3d_reader_next_serials": (_i, [_p, _p, _i, C.c_uint64, _i, _p, _p]),
    "h3d_decode_records_gather": (_i, [_p, _i, _p, _i64, _p, _i, _i, _p, _p, _p, _p, _p]),
    "h3d_resize_frames": (_i, [_p, _p, _i, _i, _i, _i, _i, _i, _p, _p]),
    "h3d_resize_frames_fmt": (_i, [_p, _p, _i, _i, _i, _i, _i, _i, _i, _p, _p]),
    "h3d_convert_frames": (_i, [_p, _p, _i, _i, _i, _i, _p, _p]),
    "h3d_augment_image":(_i, [_p, _p, _p, _p, _i, _i, _i, _i, _i, _p, _p, _p, _p]),
    "h3d_rhd_reader_items_aug": (_i, [_p, _p, _p, _p, _i, _i, _i, _i, _p, _i, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "h3d_gaussian_scoremap_dropout": (_i, [_p, _p, _p, _p, _i, _f, _i, _i, _i, _i, _f, _p, _p]),
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
    "h3d_rotate_canonical_backward": (_i, [_p, _p, _p, _p, _p, _p, _i, _p, _p, _p]),
    "h3d_bone_rel_trafo_inv_backward": (_i, [_p, _p, _p, _p, _i, _p]),
    "h3d_bone_rel_trafo": (_i, [_p, _p, _p, _i, _p]),
    "h3d_mse_loss_forward": (_i, [_p, _p, _p, _i64, _p, _p]),
    "h3d_mse_loss_backward": (_i, [_p, _p, _p, _p, _i64, _p, _p]),
    "h3d_eval_store_bytes": (_i64, [_i, _i, _i]),
    "h3d_eval_feed": (_i, [_p, _p, _i, _i, _i, _p, _p, _p, _i, _i, _p]),
    "h3d_eval_stats": (_i, [_p, _p, _i, _i, _i, _p, _i, _p, _p]),
    "h3d_draw_segments": (_i, [_p, _p, _i, _i, _i, _p, _i, _p, _p, _f, _p]),
    "h3d_set_dropout": (_i, [_p, _i, C.c_uint64]),
    "h3d_dropout_draw": (_i, [_p, C.POINTER(_p)]),
    "h3d_dropout_forward": (_i, [_p, _p, _i, _i, _f, _i, _p, _p, _p]),
    "h3d_dropout_forward_planes": (_i, [_p, _p, _i, _i, _f, _i, _p, _p, _i, _i, _p, _p, _p]),
    "h3d_dropout_backward": (_i, [_p, _p, _p, _i, _i, _f, _p, _p]),
    "h3d_dropout_advance": (_i, [_p, _p]),
}
# the camera-rig entries (include/hand3d_b200_rig.h, included by hand3d_b200.h), bound by load() like the ones above; their launch
# counts are checked against the profiler by tests/test_gpu_frames_rig.py
RIG_SIGNATURES = {
    "h3d_frame_rig_query": (_i, [_i, _p, _p, _i, _i, _p, C.POINTER(_i64), _p, C.POINTER(_i64)]),
    "h3d_frame_rig_plan": (_i, [_p, _i, _p, _p, _i, _i, _p]),
    "h3d_resize_frames_rig": (_i, [_p, _p, _i, _p, _p, _i, _i, _i, _p, _p]),
}
ADAM_STATE_WORDS = 4   # H3D_ADAM_STATE_WORDS
# training-mode reader augmentation (H3D_AUG_*): flags, and the per-sample parameter layout
AUG_COORD_UV_NOISE, AUG_CROP_CENTER_NOISE, AUG_CROP_SCALE_NOISE, AUG_CROP_OFFSET_NOISE, AUG_HUE, AUG_RANDOM_CROP, AUG_SCOREMAP_DROPOUT = 1, 2, 4, 8, 16, 32, 64
AUG_STREAM_ITEMS, AUG_STREAM_SHUFFLE, AUG_MAX_ATTEMPTS = 0, 1, 16
AUG_UV_NOISE, AUG_CENTER_NOISE, AUG_SCALE, AUG_OFFSET_NOISE, AUG_HUE_DELTA, AUG_WINDOW, AUG_KEEP, AUG_USED, AUG_PARAMS = 0, 84, 86, 87, 89, 90, 92, 113, 128
# device-resident reading (H3D_READER_*): the queue state layout and the largest gather
READER_QUEUE_CAPACITY, READER_STATE_COUNT, READER_STATE_NEXT, READER_STATE_SLOTS, READER_STATE_WORDS, READER_MAX_GATHER = 100, 0, 1, 2, 102, 4096
# camera frames (H3D_FRAME_*): the largest frame side and output side of h3d_resize_frames
FRAME_MAX_SIDE, FRAME_MAX_OUT = 4096, 512
# pixel formats of camera frames (H3D_PIXEL_*), by the names hand3d_b200.frames takes
PIXEL_FORMATS = {"rgb": 0, "bgr": 1, "nv12": 2, "i420": 3, "yuyv": 4}
# camera rigs (H3D_FRAME_RIG_*, H3D_RIG_*): the most slots, and the layout of h3d_frame_rig_query's table
FRAME_RIG_MAX_SLOTS, FRAME_RIG_SLOT_WORDS, FRAME_RIG_LAUNCH_WORDS = 64, 24, 4
RIG_FORMAT, RIG_H, RIG_W, RIG_KXS, RIG_KYS, RIG_BAND, RIG_CHUNK, RIG_ROW_STRIDE, RIG_NBANDS = 0, 1, 2, 3, 4, 5, 6, 7, 8
RIG_ACC_BYTES, RIG_INTER_BYTES, RIG_SMEM, RIG_SEG_OFF, RIG_RGB_STRIDE, RIG_XB, RIG_KX, RIG_YB, RIG_KY, RIG_CTA0, RIG_SIZE = 9, 10, 11, 12, 15, 16, 17, 18, 19, 20, 21
RIG_LAUNCH_FIRST, RIG_LAUNCH_SLOTS, RIG_LAUNCH_CTAS, RIG_LAUNCH_SMEM = 0, 1, 2, 3
# the largest image side of h3d_pipeline_forward and h3d_seg_postprocess (H3D_PIPELINE_MAX_SIDE)
PIPELINE_MAX_SIDE = 2048
# tracking state (H3D_TRACK_*): the word offset of each array, in units of B words
TRACK_CENTER, TRACK_SCALE, TRACK_SCORE, TRACK_LOST, TRACK_STATE_WORDS = 0, 2, 3, 4, 5
# device evaluation store (H3D_EVAL_*): dtypes, the header layout, the limits and the layout of a stats row
EVAL_FLOAT32, EVAL_FLOAT64 = 0, 1
EVAL_KEPT, EVAL_DROPPED, EVAL_TICKET, EVAL_COUNT, EVAL_HEADER_WORDS = 0, 1, 2, 8, 72
EVAL_MAX_KP, EVAL_MAX_DIM, EVAL_MAX_SAMPLES, EVAL_MAX_THRESHOLDS = 64, 4, 1 << 24, 4096
EVAL_STAT_N, EVAL_STAT_MEAN, EVAL_STAT_MEDIAN, EVAL_STAT_COUNTS = 0, 1, 2, 3
# drawing (H3D_DRAW_*): the most segments per call and the widest line of h3d_draw_segments
DRAW_MAX_SEGMENTS, DRAW_MAX_LINEWIDTH = 64, 64
# dropout of the lifting stage (H3D_DROPOUT_*): the generator's stream id, the layer ids and their keep probabilities
DROPOUT_STREAM = 2
DROPOUT_LAYER_FC_REL0, DROPOUT_LAYER_FC_REL1, DROPOUT_LAYER_FC_VP0, DROPOUT_LAYER_FC_VP1, DROPOUT_LAYER_OP = 0, 1, 2, 3, 4
DROPOUT_KEEP_POSEPRIOR, DROPOUT_KEEP_VIEWPOINT = 0.8, 0.75

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
    for name, (res, args) in list(SIGNATURES.items()) + list(RIG_SIGNATURES.items()):
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

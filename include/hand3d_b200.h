/*
 * hand3d_b200 -- C ABI of the H100-native ColorHandPose3D forward pass.
 *
 * The reference (lmb-freiburg/hand3d) has no FFI boundary: its hot path sits behind the Python API
 * of nets/ColorHandPose3DNetwork.py / nets/PosePriorNetwork.py / utils/general.py and resolves to
 * TensorFlow-1.3 library kernels.  This header is the boundary a maintainer binds instead (ctypes
 * stub in INTEGRATION.md); every entry point cites the reference interface it replaces.
 *
 * Conventions (SURVEY.md 8b):
 *   - plain C, raw DEVICE pointers unless a parameter is named host_*, explicit sizes, NHWC fp32
 *     tensors exactly as the reference lays them out;
 *   - every compute call ENQUEUES work on `stream` (a cudaStream_t passed as void*) and returns at once: no device
 *     synchronisation, no per-call cudaMalloc / cudaFree (capturable into a CUDA graph).  The caller owns all tensors and the
 *     workspace arena of the stage entry points; operator entry points borrow scratch from a context-owned buffer that only
 *     ever grows (old blocks are retired until h3d_destroy), so consecutive operator calls on one context must be ordered by
 *     the caller when they run on different streams.  Documented exceptions: h3d_load_weight, h3d_pack_conv_weights and the
 *     host-weight convenience entry h3d_conv2d_tc(_strided) upload weights (allocate + copy);
 *   - return 0 on success, negative H3D_E* on failure; h3d_last_error() gives a thread-local message;
 *   - one h3d_ctx per device, used from one host thread at a time (one rank <-> one GPU); every entry makes the context's device
 *     current for the duration of the call and restores the caller's device;
 *   - there is NO CPU fallback: without a usable sm_90a device every compute call fails with
 *     H3D_ENODEVICE.
 */
#ifndef HAND3D_B200_H_
#define HAND3D_B200_H_

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define H3D_API __attribute__((visibility("default")))
#else
#define H3D_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define H3D_OK 0
#define H3D_EINVAL (-1)     /* bad argument / shape                                   */
#define H3D_ENODEVICE (-2)  /* no CUDA device, or not compute capability 10.x          */
#define H3D_ECUDA (-3)      /* CUDA runtime / driver error (message in h3d_last_error) */
#define H3D_EWEIGHTS (-4)   /* weights missing, unknown name, wrong shape, NaN/Inf     */
#define H3D_EWORKSPACE (-5) /* workspace arena missing or too small                    */

/* Arithmetic of the tensor-core convolution layers. */
#define H3D_PREC_FP32_FFMA 0  /* all layers on CUDA cores in fp32 (validation yard-stick)             */
#define H3D_PREC_BF16X3 1     /* wgmma,   bf16 hi/lo split, 3 MMA passes, fp32 accumulate (fp32 parity) */
#define H3D_PREC_FP16X3 2     /* wgmma,   fp16 hi/lo split, 3 MMA passes, fp32 accumulate (fp32 parity for activations of
                                 magnitude 2^-6 .. 2^10 of unit scale; weights carry a per-channel power-of-two shift) */
#define H3D_PREC_FP16 3       /* wgmma,   fp16 single pass, fp32 accumulate (BASELINE config 5, 1e-2)   */
#define H3D_PREC_BF16 4       /* wgmma,   bf16 single pass                                              */
#define H3D_PREC_FP16_F8C 5   /* wgmma,   fp16 main pass + two fp8 (e4m3) correction passes, fp32 accumulate.  fp32 grade (scale-relative
                                 error 4.4e-6 measured on an H100 80GB HBM3 at 400 W) only inside its range: activations 2^-2 .. 2^6 of
                                 unit scale and a layer's largest |w| >= ~2.5e-3; outside it degrades towards fp16 grade unreported,
                                 and |x| >= 2047 saturates the fp16 main plane (DESIGN.md section 6.1) */

/* PosePriorNetwork variants (nets/PosePriorNetwork.py:64-93). */
#define H3D_VARIANT_DIRECT 0
#define H3D_VARIANT_BOTTLENECK 1
#define H3D_VARIANT_PROPOSED 2
#define H3D_VARIANT_LOCAL 3 /* 'local' and 'local_w_xyz_loss': direct prediction of bone-relative coords + bone_rel_trafo_inv */

typedef struct h3d_ctx h3d_ctx;

H3D_API const char* h3d_last_error(void);
H3D_API int h3d_version(void);
/* 1 when a CUDA device with compute capability 10.x is visible, else 0 (never fails). */
H3D_API int h3d_device_available(void);

/* ---- context ----------------------------------------------------------------------------- */
H3D_API int h3d_create(h3d_ctx** out, int device);
H3D_API int h3d_destroy(h3d_ctx* ctx);
H3D_API int h3d_set_precision(h3d_ctx* ctx, int precision);
H3D_API int h3d_get_precision(const h3d_ctx* ctx);
/* Kernel-selection switches for A/B measurements and forced-variant tests (process-wide; initialised ONCE from the H3D_*
 * environment variables when the library is first used, never read on a launch path).  Keys: "tc_2cta" (-1 policy / 0 / 1),
 * "tc_bn" (0 policy / 64 / 128), "tc_c64", "tc_c64x2", "tc_pair128", "tc_stack", "tc_chunk_kb", "no_side_stream",
 * "no_pool_fusion", "lift_direct", "c3_ffma", "c3_tma", "pdl", "fc_chain", "c64_tma_out", "tc_chain", "tc_small_split", "fuse_c1",
 * "no_seg_fusion".  "tc_2cta", "tc_c64", "tc_c64x2", "tc_pair128", "tc_stack", "c3_tma", "c64_tma_out", "tc_chain", "tc_small_split"
 * and "fuse_c1" select nothing in the sm_90a build (one convolution kernel family) and are accepted for compatibility.
 * ctx may be NULL; when given, its cached layer plans are dropped (never while a CUDA graph captured from this context is alive:
 * graphs hold plan-owned pointers). */
H3D_API int h3d_set_tuning(h3d_ctx* ctx, const char* key, int value);
/* Device-side error word (pinned host memory, survives a trapped kernel): 0 = none; 1-5 = a bounded mbarrier wait of a tensor-core
 * convolution kernel timed out (1 TMA producer waiting for a free stage, 3 wgmma warpgroup waiting for a loaded stage) and the
 * kernel trapped; 100 + r = h3d_gather_records_p2p
 * never saw peer rank r's records.  Returns H3D_OK or H3D_ECUDA (message in h3d_last_error); *code (optional) = the word. */
H3D_API int h3d_check_errors(h3d_ctx* ctx, int* code);
/* Number of kernels this library launched through `ctx` since creation (bench "gpu_launches"). */
H3D_API int64_t h3d_launch_count(const h3d_ctx* ctx);

/* Per-kernel-class device timing for bench.py's roofline: between begin and end every plan step is
 * bracketed by CUDA events on its launch stream.  Classes: 0 = tensor-core conv, 1 = CUDA-core conv,
 * 2 = fully connected, 3 = other.  end() synchronises and fills three arrays of length 4. */
H3D_API int h3d_profile_begin(h3d_ctx* ctx);
H3D_API int h3d_profile_end(h3d_ctx* ctx, double* ms_by_kind, int64_t* flops_by_kind, int64_t* launches_by_kind);

/* Replaces ColorHandPose3DNetwork.init / PosePriorNetwork.init (nets/ColorHandPose3DNetwork.py:34-59,
 * nets/PosePriorNetwork.py:36-57): one call per pickled variable, `name` = "<scope>/<layer>/weights|biases",
 * host_data = fp32 HWIO / [in,out] / [Cout] exactly as pickled.  Unknown names and wrong shapes fail
 * (assign_from_values behaviour); FC weights/biases containing NaN/Inf fail (tf.check_numerics,
 * utils/general.py:122,127).  Weights are packed once to the kernel layouts. */
H3D_API int h3d_load_weight(h3d_ctx* ctx, const char* name, const float* host_data, const int64_t* shape, int ndim);
/* 1 if every variable of `scope` ("HandSegNet", "PoseNet2D", "PosePrior", "ViewpointNet") is loaded. */
H3D_API int h3d_scope_ready(const h3d_ctx* ctx, const char* scope);

/* Workspace arena for the stage entry points (activations of one batch). */
H3D_API int64_t h3d_workspace_bytes(const h3d_ctx* ctx, int B, int H, int W);
H3D_API int h3d_set_workspace(h3d_ctx* ctx, void* dev_ptr, int64_t bytes);

/* ---- stage entry points (fixed layer schedules) --------------------------------------------- */
/* ColorHandPose3DNetwork.inference_detection (nets/ColorHandPose3DNetwork.py:131-168).
 * image [B,H,W,3] -> logits [B,H,W,2] (already x8 bilinearly up-sampled, TF1 legacy resize). */
H3D_API int h3d_handsegnet_forward(h3d_ctx* ctx, const float* image, int B, int H, int W, float* logits, void* stream);

/* ColorHandPose3DNetwork.inference_pose2d (nets/ColorHandPose3DNetwork.py:170-219).
 * image_crop [B,Hc,Wc,3] (Hc,Wc multiples of 8) -> s0,s1,s2 [B,Hc/8,Wc/8,21] (any may be NULL). */
H3D_API int h3d_posenet_forward(h3d_ctx* ctx, const float* image_crop, int B, int Hc, int Wc,
                        float* s0, float* s1, float* s2, void* stream);

/* ColorHandPose3DNetwork._inference_pose3d (nets/ColorHandPose3DNetwork.py:221-247) and the
 * PosePriorNetwork variants (nets/PosePriorNetwork.py:64-93, H3D_VARIANT_*).
 * scoremap [B,32,32,21], hand_side [B,2] -> coord_xyz_rel_normed [B,21,3]; optional coord_can [B,21,3],
 * rot_mat [B,3,3] (NULL to skip; rot_mat is only written for H3D_VARIANT_PROPOSED). */
H3D_API int h3d_lifting_forward(h3d_ctx* ctx, const float* scoremap32, const float* hand_side, int B, int variant,
                        float* coord_xyz_rel_normed, float* coord_can, float* rot_mat, void* stream);

/* ColorHandPose3DNetwork.inference / inference2d (nets/ColorHandPose3DNetwork.py:61-129), plus
 * detect_keypoints (utils/general.py:331-344) on device.  with_pose3d == 0 -> inference2d (hand_side,
 * keypoint_coord3d may be NULL).  force_center/force_scale non-NULL: teacher-forced crop parameters.
 * Outputs (device, caller-owned, any of the large ones may be NULL to skip the copy-out):
 *   hand_scoremap [B,H,W,2], image_crop [B,256,256,3], scale_crop [B,1], center [B,2],
 *   keypoints_scoremap [B,256,256,21], keypoint_coord3d [B,21,3], keypoints_uv [B,21,2] int32 (row,col),
 *   hand_mask [B,H,W] uint8 (optional). */
H3D_API int h3d_pipeline_forward(h3d_ctx* ctx, const float* image, const float* hand_side, int B, int H, int W,
                         int with_pose3d, const float* force_center, const float* force_scale,
                         float* hand_scoremap, float* image_crop, float* scale_crop, float* center,
                         float* keypoints_scoremap, float* keypoint_coord3d, int32_t* keypoints_uv,
                         uint8_t* hand_mask, void* stream);

/* ColorHandPose3DNetwork.inference_pose2d + the x8 up-sampling and key-point detection of eval2d_gt_cropped.py:45-50,78:
 * image_crop [B,Hc,Wc,3] -> keypoints_scoremap [B,Hc,Wc,21] (tf.image.resize_images of the last stage; may be NULL when
 * Hc, Wc <= 256: kept in the workspace) and keypoints_uv [B,21,2] int32 (row, col) (may be NULL). */
H3D_API int h3d_pose2d_forward(h3d_ctx* ctx, const float* image_crop, int B, int Hc, int Wc, float* keypoints_scoremap,
                               int32_t* keypoints_uv, void* stream);

/* ---- operator entry points (utils/general.py) ------------------------------------------------- */
/* NetworkOps.conv / conv_relu (utils/general.py:36-59): tf.nn.conv2d SAME + bias (+ leaky 0.01).
 * fp32 CUDA-core kernel; x [B,H,W,Cin], w HWIO [k,k,Cin,Cout] (device), y [B,ceil(H/s),ceil(W/s),Cout]. */
H3D_API int h3d_conv2d_f32(h3d_ctx* ctx, const float* x, const float* w_hwio, const float* bias, float* y,
                   int B, int H, int W, int Cin, int Cout, int ksize, int stride, int leaky, void* stream);
/* Same op on the wgmma tensor-core path (stride 1, Cin and Cout multiples of 64 after internal padding;
 * ksize in {1,3,5,7}); host_w_hwio / host_bias are HOST pointers: this convenience entry packs, uploads and frees the weights
 * around the call (allocates, and the free waits for the kernel) -- use h3d_pack_conv_weights + h3d_conv2d_tc_packed on a hot path. */
H3D_API int h3d_conv2d_tc(h3d_ctx* ctx, const float* x, const float* host_w_hwio, const float* host_bias, float* y,
                  int B, int H, int W, int Cin, int Cout, int ksize, int leaky, int precision, void* stream);
/* Same with the `stride` argument of NetworkOps.conv (utils/general.py:36-53): 1, or 2 with even H and W and ksize >= 3 (the lifting
 * pyramids, nets/ColorHandPose3DNetwork.py:255-258,291-294); y [B,H/stride,W/stride,Cout].  TF 'SAME' pads 0 before / 1 after
 * for stride 2 on an even size, i.e. the result is the stride-1 output at the odd pixels. */
H3D_API int h3d_conv2d_tc_strided(h3d_ctx* ctx, const float* x, const float* host_w_hwio, const float* host_bias, float* y,
                          int B, int H, int W, int Cin, int Cout, int ksize, int stride, int leaky, int precision, void* stream);
/* Enqueue-only form of the tensor-core convolution: weights packed once (HOST pointers, HWIO / [Cout]) into a handle ... */
typedef struct h3d_packed_conv h3d_packed_conv;
H3D_API int h3d_pack_conv_weights(h3d_ctx* ctx, const float* host_w_hwio, const float* host_bias, int ksize, int Cin, int Cout,
                                  int precision, h3d_packed_conv** out);
H3D_API int h3d_free_packed_conv(h3d_ctx* ctx, h3d_packed_conv* packed);
/* ... and applied any number of times: x [B,H,W,Cin] -> y [B,H/stride,W/stride,Cout]; operand planes live in the context's
 * operator scratch (no allocation, no synchronisation). */
H3D_API int h3d_conv2d_tc_packed(h3d_ctx* ctx, const float* x, const h3d_packed_conv* packed, float* y, int B, int H, int W,
                                 int stride, int leaky, void* stream);
/* The same forward with DEVICE weights (w_hwio [k,k,Cin,Cout], bias [Cout]), for weights that change every optimiser step: a kernel
 * packs them into the context's operator scratch, so the call only enqueues work.  Bit-identical to h3d_pack_conv_weights +
 * h3d_conv2d_tc_packed for the same weights.  precision: bf16x3, fp16x3, fp16 or bf16. */
H3D_API int h3d_conv2d_tc_dev(h3d_ctx* ctx, const float* x, const float* w_hwio, const float* bias, float* y, int B, int H, int W,
                              int Cin, int Cout, int ksize, int stride, int leaky, int precision, void* stream);
/* Gradients of y = act(conv_SAME(x, w, stride) + b) (act: identity, or leaky ReLU 0.01 when leaky), the TF Conv2DBackpropInput,
 * Conv2DBackpropFilter, BiasAddGrad and Maximum gradients that AdamOptimizer.minimize evaluates (training_posenet.py:67,
 * training_handsegnet.py).  x [B,H,W,Cin], y and dy [B,H/stride,W/stride,Cout], w_hwio [k,k,Cin,Cout], all fp32 device tensors;
 * outputs dx [B,H,W,Cin], dw_hwio [k,k,Cin,Cout], db [Cout], each may be NULL to skip it (a first layer needs no dx).  y is required
 * with leaky (the slope is chosen where y >= 0, as TF's Maximum gradient does), x with dw_hwio, w_hwio with dx.  Same geometry as
 * h3d_conv2d_tc_strided, Cout <= 1024; precision bf16x3 (fp32 parity) or bf16, the fp16 modes return H3D_EINVAL.  Enqueue-only
 * (operator scratch), deterministic bit for bit; capturable into a CUDA graph once a first call has sized the scratch. */
H3D_API int h3d_conv2d_tc_backward(h3d_ctx* ctx, const float* x, const float* y, const float* dy, const float* w_hwio, float* dx,
                                   float* dw_hwio, float* db, int B, int H, int W, int Cin, int Cout, int ksize, int stride, int leaky,
                                   int precision, void* stream);
/* NetworkOps.leaky_relu (utils/general.py:31-33): y = max(x, 0.01 x), n elements, 16-byte aligned pointers. */
H3D_API int h3d_leaky_relu_f32(h3d_ctx* ctx, const float* x, float* y, int64_t n, void* stream);
/* NetworkOps.max_pool (utils/general.py:62-65): 2x2 / 2 VALID. */
H3D_API int h3d_maxpool2x2_f32(h3d_ctx* ctx, const float* x, float* y, int B, int H, int W, int C, void* stream);
/* Gradient of NetworkOps.max_pool (TF MaxPoolGrad under AdamOptimizer.minimize, training_posenet.py:67): x [B,H,W,C] (the forward
 * input), dy [B,H/2,W/2,C] -> dx [B,H,W,C]; each window's gradient goes to its first maximum in row-major order, as TF's CPU kernel. */
H3D_API int h3d_maxpool2x2_backward_f32(h3d_ctx* ctx, const float* x, const float* dy, float* dx, int B, int H, int W, int C, void* stream);
/* NetworkOps.fully_connected(_relu) (utils/general.py:113-136): y = x[B,in] @ w[in,out] + b. */
H3D_API int h3d_fully_connected_f32(h3d_ctx* ctx, const float* x, const float* w, const float* bias, float* y,
                            int B, int in_features, int out_features, int leaky, void* stream);
/* tf.image.resize_images bilinear, align_corners=False, TF1 legacy (nets/...:97,128,166). */
H3D_API int h3d_resize_bilinear_tf1(h3d_ctx* ctx, const float* x, float* y, int B, int H, int W, int C,
                            int out_h, int out_w, void* stream);
/* tf.nn.avg_pool 8x8/8 (nets/PosePriorNetwork.py:61). */
H3D_API int h3d_avgpool8(h3d_ctx* ctx, const float* x, float* y, int B, int H, int W, int C, void* stream);
/* single_obj_scoremap + calc_center_bb + crop-scale glue (utils/general.py:233-328,
 * nets/ColorHandPose3DNetwork.py:83-85).  logits [B,H,W,2] -> hand_mask [B,H,W] uint8 (optional),
 * max_loc [B,2] int32 (optional, find_max_location), center [B,2], crop_size [B,1] (raw, optional),
 * scale_crop [B,1].  H,W <= 512, W % 32 == 0 not required. */
H3D_API int h3d_seg_postprocess(h3d_ctx* ctx, const float* logits, int B, int H, int W, uint8_t* hand_mask,
                        int32_t* max_loc, float* center, float* crop_size, float* scale_crop, void* stream);
/* calc_center_bb (utils/general.py:271-328) on an arbitrary mask [B,H,W] fp32 (pixels with int(mask) == 1 count):
 * center [B,2] (row, col), bb [B,2,2] = [[x_min, x_max], [y_min, y_max]] (optional), crop_size [B,1] (optional); an empty mask
 * gives center (160, 160), crop_size 100, bb (+inf, -inf) as the reference's tf.cond fall-backs do. */
H3D_API int h3d_calc_center_bb(h3d_ctx* ctx, const float* mask, int B, int H, int W, float* center, float* bb, float* crop_size,
                               void* stream);
/* crop_image_from_xy (utils/general.py:163-196) incl. tf.image.crop_and_resize bilinear/extrapolation 0. */
H3D_API int h3d_crop_image_from_xy(h3d_ctx* ctx, const float* image, const float* center, const float* scale,
                           float* image_crop, int B, int H, int W, int C, int crop_size, void* stream);
/* detect_keypoints (utils/general.py:331-344), batched: scoremaps [B,H,W,C] -> [B,C,2] int32 (row,col),
 * first occurrence of the maximum in row-major order. */
H3D_API int h3d_detect_keypoints(h3d_ctx* ctx, const float* scoremaps, int B, int H, int W, int C,
                         int32_t* keypoints_uv, void* stream);
/* tf.image.resize_images (nets/ColorHandPose3DNetwork.py:96-97) fused with detect_keypoints: 21-channel score maps [B,H,W,21] ->
 * scoremaps_up [B,out_h,out_w,21] and keypoints_uv [B,21,2] int32 (row, col) of the up-sampled maps in one pass. */
H3D_API int h3d_upsample_detect_keypoints(h3d_ctx* ctx, const float* scoremaps, int B, int H, int W, int out_h, int out_w,
                                          float* scoremaps_up, int32_t* keypoints_uv, void* stream);
/* Per-image result record (SURVEY.md 8(e)): coord3d [21,3] | keypoints_uv [21,2] i32 (bit-cast) | center [2] | scale_crop [1]
 * = 108 words = 432 B.  records [B,108]. */
H3D_API int h3d_pack_records(h3d_ctx* ctx, const float* coord3d, const int32_t* keypoints_uv, const float* center,
                             const float* scale_crop, int B, float* records, void* stream);
/* Multi-GPU result exchange (SURVEY.md 8(e); the reference has no multi-GPU code): packs this rank's records and all-gathers
 * them over NVLink peer memory in ONE kernel.  peer_buffers / peer_signals are DEVICE arrays of `world` device pointers: the
 * symmetric gather buffers ([2 parities][world][max_batch][108] floats each, parity_stride_floats >= world*max_batch*108) and
 * DEDICATED uint32 signal words (>= world entries, zero-initialised, used by nothing else) of all ranks, e.g. two
 * torch.distributed._symmetric_memory allocations.  Rank r's B <= max_batch records land in slot r (offset r*max_batch*108) of
 * every rank's buffer, so ranks may hold different B.  multicast_ptr: NVSwitch multicast address of the gather buffer or 0.
 * epoch must increase by 1 per call (start at 1).  On completion (stream order) the local buffer's parity (epoch & 1) holds all
 * ranks' slots.  A peer that never signals (~10 s) sets the context's error word (h3d_check_errors) instead of hanging. */
H3D_API int h3d_gather_records_p2p(h3d_ctx* ctx, const float* coord3d, const int32_t* keypoints_uv, const float* center,
                                   const float* scale_crop, int B, int max_batch, const uint64_t* peer_buffers,
                                   const uint64_t* peer_signals, uint64_t multicast_ptr, int rank, int world, uint32_t epoch,
                                   int64_t parity_stride_floats, void* stream);
/* On-device decode of the dataset readers' fixed-length records (SURVEY.md 8(f) row 2).  dataset 0 = RHD
 * (data/BinaryDbReader.py:103-208; 410520-byte records: header [B,219] = 42x3 xyz | 42x2 uv | 3x3 K, image [B,320,320,3],
 * mask [B,320,320] u8, visibility [B,42] u8), dataset 1 = STB (data/BinaryDbReaderSTB.py:99-185; 922104-byte records:
 * header [B,126] = 21x3 xyz | 21x3 (u,v,valid), image [B,480/step,640/step,3]; eval_full.py:50 uses step 2).
 * image = u8 / 255 - 0.5 exactly as the readers compute it; header / mask / visibility may be NULL. */
#define H3D_DATASET_RHD 0
#define H3D_DATASET_STB 1
H3D_API int h3d_decode_records(h3d_ctx* ctx, int dataset, const uint8_t* records, int B, int step, float* header, float* image,
                               uint8_t* mask, uint8_t* visibility, void* stream);
/* The readers' DERIVED items (SURVEY.md 8(f) row 4), evaluation mode (no augmentation noise).  RHD (data/BinaryDbReader.py:139-162
 * palm substitution when use_wrist_coord == 0, :210-250 dominant hand by part-mask pixel counts / 21-key-point subsets /
 * root-relative normalisation, :269-346 ground-truth hand crop when hand_crop != 0): inputs are the outputs of h3d_decode_records
 * (header [B,219], mask = hand_parts [B,320,320] u8, visibility [B,42] u8).  Outputs (any may be NULL except hand_side):
 * keypoint_xyz21 [B,21,3], keypoint_uv21 [B,21,2] (crop space when hand_crop), keypoint_vis21 [B,21] u8, hand_side [B,2] one-hot,
 * keypoint_scale [B], keypoint_xyz21_normed [B,21,3], crop_center [B,2] (row, col) and crop_scale [B] (feed h3d_crop_image_from_xy
 * to obtain image_crop), cam_mat [B,3,3] (updated for the crop when hand_crop). */
H3D_API int h3d_rhd_reader_items(h3d_ctx* ctx, const float* header, const uint8_t* hand_parts, const uint8_t* visibility, int B,
                                 int use_wrist_coord, int hand_crop, int crop_size, float* keypoint_xyz21, float* keypoint_uv21,
                                 uint8_t* keypoint_vis21, float* hand_side, float* keypoint_scale, float* keypoint_xyz21_normed,
                                 float* crop_center, float* crop_scale, float* cam_mat, void* stream);
/* STB (data/BinaryDbReaderSTB.py:123-196): header [B,126] -> metres, convert_kp order (:397-410), wrist extrapolation when
 * use_wrist_coord != 0, root-relative normalisation.  hand_side is the constant (1, 0) for this dataset. */
H3D_API int h3d_stb_reader_items(h3d_ctx* ctx, const float* header, int B, int use_wrist_coord, float* keypoint_xyz21, float* keypoint_uv21,
                                 uint8_t* keypoint_vis21, float* keypoint_scale, float* keypoint_xyz21_normed, void* stream);
/* create_multiple_gaussian_map (data/BinaryDbReader.py:413-459): coords_hw [B,N,2] (row, col; truncated to int32), valid [B,N] u8
 * (NULL = all valid) -> scoremap [B,H,W,N] = exp(-d^2 / sigma^2) for key-points strictly inside the map, 0 otherwise.  N <= 64. */
H3D_API int h3d_gaussian_scoremap(h3d_ctx* ctx, const float* coords_hw, const uint8_t* valid, int B, int N, int H, int W, float sigma,
                                  float* scoremap, void* stream);
/* canonical_trafo (+ flip_right_hand, + the tf.matrix_inverse the readers apply) (utils/canonical_trafo.py:97-162,
 * data/BinaryDbReader.py:247-252): coords_xyz [B,21,3] -> coords_can [B,21,3] (z mirrored where cond_right[b] != 0; cond_right may be
 * NULL), rot_mat [B,3,3] (total rotation), rot_mat_inv [B,3,3]; each output may be NULL. */
H3D_API int h3d_canonical_trafo(h3d_ctx* ctx, const float* coords_xyz, const uint8_t* cond_right, int B, float* coords_can, float* rot_mat,
                                float* rot_mat_inv, void* stream);
/* EvalUtil.feed (utils/general.py:531-549), batched on device: gt / pred [n, D] (D = 2 or 3), vis [n] u8 ->
 * dist [n] = ||gt - pred||_2, or -1 where the key-point is not visible. */
H3D_API int h3d_eval_keypoint_dist(h3d_ctx* ctx, const float* gt, const uint8_t* vis, const float* pred, int n, int D, float* dist,
                                   void* stream);
/* bone_rel_trafo_inv (utils/relative_trafo.py:243-295): coords_rel [B,21,3] (length, angle_x, angle_y) -> xyz [B,21,3]. */
H3D_API int h3d_bone_rel_trafo_inv(h3d_ctx* ctx, const float* coords_rel, float* coords_xyz, int B, void* stream);
/* _get_rot_mat + _flip_right_hand + matmul (nets/ColorHandPose3DNetwork.py:239-247,311-384). */
H3D_API int h3d_rotate_canonical(h3d_ctx* ctx, const float* coord_can, const float* uxyz, const float* hand_side,
                         int B, float* rot_mat, float* coord_out, void* stream);
/* _flip_right_hand (nets/ColorHandPose3DNetwork.py:336-361): out = coords with z negated where cond_right[b] != 0 (u8 [B]). */
H3D_API int h3d_flip_right_hand(h3d_ctx* ctx, const float* coords_xyz, const uint8_t* cond_right, int B, float* out, void* stream);

/* ---- Training of HandSegNet and PoseNet2D (training_posenet.py, training_handsegnet.py) ----
 * Like h3d_conv2d_tc_backward: enqueue-only (operator scratch), no float atomics, every sum in an order fixed by the shapes, so the
 * results are bit-reproducible; capturable into a CUDA graph once a first call has sized the scratch.  grad_loss is the incoming
 * gradient of a loss as a DEVICE scalar (NULL = 1), so a backward never reads a value on the host. */

/* Gradient of tf.image.resize_images (TF ResizeBilinearGrad: bilinear, align_corners = False, TF1 legacy) between the networks and
 * their losses (training_posenet.py:49, nets/ColorHandPose3DNetwork.py:166): dy [B,out_h,out_w,C] -> dx [B,H,W,C], the exact adjoint
 * of h3d_resize_bilinear_tf1 (source indices and weights from the forward's own fp32 operations), any ratio, up or down; equal sizes
 * copy.  Sums gather in ascending output order. */
H3D_API int h3d_resize_bilinear_tf1_backward(h3d_ctx* ctx, const float* dy, float* dx, int B, int H, int W, int C, int out_h, int out_w,
                                             void* stream);
/* PoseNet score-map loss for one predicted map (training_posenet.py:58-61):
 *   loss = sum_{b,k} vis[b,k] sqrt(mean_{h,w} (pred - target)^2) / (sum_{b,k} vis + 0.001)
 * pred, target [B,H,W,21], vis [B,21] fp32 (0 / 1, any value is accepted) -> loss (device scalar) and rms [B,21] =
 * sqrt(mean (pred - target)^2), which the backward reuses.  fp32 with separate multiply and add. */
H3D_API int h3d_scoremap_loss_forward(h3d_ctx* ctx, const float* pred, const float* target, const float* vis, int B, int H, int W,
                                      float* loss, float* rms, void* stream);
/* Its gradient: dpred [B,H,W,21] = grad_loss vis[b,k] / S (pred - target) / (H W rms[b,k]), S = sum vis + 0.001; 0 where
 * rms[b,k] == 0 (TF's SqrtGrad gives NaN there). */
H3D_API int h3d_scoremap_loss_backward(h3d_ctx* ctx, const float* pred, const float* target, const float* vis, const float* rms,
                                       const float* grad_loss, int B, int H, int W, float* dpred, void* stream);
/* HandSegNet loss (training_handsegnet.py:56-60): reduce_mean(softmax_cross_entropy_with_logits(logits, labels)) over `rows` rows of 2
 * classes.  logits, labels [rows,2] fp32 (8-byte aligned; labels need not be one-hot) -> loss (device scalar).  Per row as TF's
 * SoftmaxXentWithLogits: m = max, s = sum exp(x - m), loss = sum labels (log s - (x - m)). */
H3D_API int h3d_softmax_xent_forward(h3d_ctx* ctx, const float* logits, const float* labels, int64_t rows, float* loss, void* stream);
/* Its gradient: dlogits [rows,2] = grad_loss / rows (softmax(logits) - labels). */
H3D_API int h3d_softmax_xent_backward(h3d_ctx* ctx, const float* logits, const float* labels, const float* grad_loss, int64_t rows,
                                      float* dlogits, void* stream);

/* tf.train.AdamOptimizer (TF 1.3 ApplyAdam, training_posenet.py:67).  The optimiser state is H3D_ADAM_STATE_WORDS 32-bit words of
 * DEVICE memory owned by the caller: [lr, beta1_power, beta2_power (fp32), ticket (uint32, 0 between steps)].  Keeping the learning
 * rate and the beta powers on the device lets a captured CUDA graph replay the step. */
#define H3D_ADAM_STATE_WORDS 4
typedef struct h3d_adam_tensor {   /* one variable: param, its gradient and the slots m, v, all fp32 [numel] device arrays */
    float* param;
    const float* grad;
    float* m;
    float* v;
    int64_t numel;
} h3d_adam_tensor;
/* Writes the state: lr, beta1_power and beta2_power (a fresh optimiser: beta1_power = beta1, beta2_power = beta2, as TF creates the
 * accumulators) and clears the ticket.  Enqueued on `stream`. */
H3D_API int h3d_adam_state_set(h3d_ctx* ctx, float* state, float lr, float beta1_power, float beta2_power, void* stream);
/* Writes the learning rate only (LearningRateScheduler.get_lr's value for this step). */
H3D_API int h3d_adam_set_lr(h3d_ctx* ctx, float* state, float lr, void* stream);
/* One Adam step over every tensor of `table` (a DEVICE array of num_tensors <= 1024 entries) in one launch.  Per element, in this order
 * and in fp32 without contraction: alpha = lr sqrt(1 - beta2_power) / (1 - beta1_power) (once per call), m += (g - m)(1 - beta1),
 * v += (g^2 - v)(1 - beta2), param -= m alpha / (sqrt(v) + epsilon): TF's epsilon-hat form, which differs from torch.optim.Adam for
 * small gradients.  After every element has used them, the last block multiplies beta1_power by beta1 and beta2_power by beta2 (fp32),
 * as AdamOptimizer._finish does.  The reference's defaults are beta1 0.9, beta2 0.999, epsilon 1e-8. */
H3D_API int h3d_adam_step(h3d_ctx* ctx, const h3d_adam_tensor* table, int num_tensors, float* state, float beta1, float beta2,
                          float epsilon, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* HAND3D_B200_H_ */

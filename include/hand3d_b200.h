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
 *     host-weight convenience entries h3d_conv2d_tc(_strided) and h3d_conv2d_layer_planes upload weights (allocate + copy);
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
#define H3D_ENODEVICE (-2)  /* no CUDA device, or not compute capability 9.0           */
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
/* 1 when a CUDA device with compute capability 9.0 is visible, else 0 (never fails). */
H3D_API int h3d_device_available(void);

/* ---- context ----------------------------------------------------------------------------- */
H3D_API int h3d_create(h3d_ctx** out, int device);
H3D_API int h3d_destroy(h3d_ctx* ctx);
H3D_API int h3d_set_precision(h3d_ctx* ctx, int precision);
H3D_API int h3d_get_precision(const h3d_ctx* ctx);
/* Kernel-selection switches for A/B measurements and forced-variant tests (process-wide; initialised ONCE from the H3D_*
 * environment variables when the library is first used, never read on a launch path).  Keys: "tc_bn" (0 policy / 64 / 128),
 * "tc_chunk_kb" (0 policy, else K blocks per partial sum), "no_side_stream", "no_pool_fusion", "lift_direct", "c3_ffma", "pdl",
 * "fc_chain", "no_seg_fusion".  Any other key returns H3D_EINVAL.
 * ctx may be NULL; when given, its cached layer plans are dropped (never while a CUDA graph captured from this context is alive:
 * graphs hold plan-owned pointers). */
H3D_API int h3d_set_tuning(h3d_ctx* ctx, const char* key, int value);
/* Device-side error word (pinned host memory, survives a trapped kernel): 0 = none; 1-5 = a bounded mbarrier wait of a tensor-core
 * convolution kernel timed out (1 TMA producer waiting for a free stage, 3 wgmma warpgroup waiting for a loaded stage) and the
 * kernel trapped; 100 + r = h3d_gather_records_p2p
 * never saw peer rank r's records.  Returns H3D_OK or H3D_ECUDA (message in h3d_last_error); *code (optional) = the word. */
H3D_API int h3d_check_errors(h3d_ctx* ctx, int* code);
/* Number of kernels this library enqueued through `ctx` since creation (bench "gpu_launches"): every kernel an entry point
 * taking `ctx` enqueues counts, kernels enqueued under stream capture included, whatever the entry returns.  Memory sets and
 * copies do not count. */
H3D_API int64_t h3d_launch_count(const h3d_ctx* ctx);

/* Per-kernel-class device timing for bench.py's roofline: between begin and end every plan step that
 * launches a kernel is bracketed by CUDA events on its launch stream.  Classes: 0 = tensor-core conv,
 * 1 = CUDA-core conv, 2 = fully connected, 3 = other.  end() synchronises and fills three arrays of
 * length 4; launches_by_kind counts the bracketed steps. */
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

/* Workspace arena for the stage entry points (activations of one batch).
 * The workspace and the context's operator scratch carry no state between calls and need no initialisation: every entry writes
 * each byte of them it reads earlier in the same call (padding channels, keys of the arg-max reductions and split-K partial sums
 * included), so any content a previous call, another context or the allocator left there never reaches a result, an address or a
 * loop bound.  State that outlives a call lives only in caller-owned buffers named as such: the Adam state, the reader queue, the
 * h3d_eval_* store and the track state. */
H3D_API int64_t h3d_workspace_bytes(const h3d_ctx* ctx, int B, int H, int W);
H3D_API int h3d_set_workspace(h3d_ctx* ctx, void* dev_ptr, int64_t bytes);
/* Fills the current operator scratch and the workspace (when one is set) with `byte` (0..255): one cudaMemsetAsync each on `stream`,
 * enqueue-only, allocates nothing, capturable.  For tests of the contract above; the scratch grows on demand, so a test sizes it with
 * one call of the entry under test before filling it. */
H3D_API int h3d_fill_scratch(h3d_ctx* ctx, int byte, void* stream);

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
 *   hand_mask [B,H,W] uint8 (optional).
 * 1 <= H, W <= H3D_PIPELINE_MAX_SIDE; a larger image returns H3D_EINVAL before anything is enqueued. */
#define H3D_PIPELINE_MAX_SIDE 2048
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

/* ---- Tracking across camera frames (extends nets/ColorHandPose3DNetwork.py:61-129 and utils/general.py:271-328,347-357) ----
 * Batch slot b is one camera stream.  A track state is caller-owned DEVICE memory of h3d_track_state_bytes(B) bytes: arrays of B x
 * 32-bit words (center takes two), the array H3D_TRACK_<name> starting at word H3D_TRACK_<name> * B:
 *   center [B,2] fp32 (row, col) and scale [B] fp32: the crop the next track step uses;
 *   score [B] fp32: (sum over k of the peak of channel k of the last PoseNet2D stage's 32x32 map) / 21 (NaN if the map holds NaN);
 *   lost [B] int32: 1 when the step's key-points were not trusted; a lost slot keeps the crop it had.
 * The caller initialises center and scale before a first track step (a detect step writes them for every slot it does not lose). */
#define H3D_TRACK_CENTER 0
#define H3D_TRACK_SCALE 2
#define H3D_TRACK_SCORE 3
#define H3D_TRACK_LOST 4
#define H3D_TRACK_STATE_WORDS 5
/* Bytes of a track state of B slots (H3D_TRACK_STATE_WORDS * 4 * B), or H3D_EINVAL for B < 1. */
H3D_API int64_t h3d_track_state_bytes(int B);
/* One step of a tracked stream.  detect != 0: h3d_pipeline_forward's computation (no forced crop, no hand_scoremap / hand_mask).
 * detect == 0: the crop (center, scale) is read from `state`, and HandSegNet, the mask post-processing and the bounding box are not
 * enqueued; the crop, PoseNet2D, the x8 up-sampling + key-point detection and the lifting stage follow as in h3d_pipeline_forward.
 * Either way the step ends with track_update_kernel, which derives the next crop from this step's key-points (fp32, round to nearest,
 * no contraction):
 *   p[k] = (float(uv[k]) - 128) / scale + center per axis; center' = 0.5 (max_k p + min_k p); size = max(extent_row, extent_col);
 *   if center' or size is not finite: center' = (160, 160), size = 100, and the slot is lost;
 *   scale' = min(max(256 / (size * margin), 0.25), 5);
 *   lost also when min_score is not NaN and !(score >= min_score).  A slot that is not lost takes (center', scale').
 * Outputs as h3d_pipeline_forward's (any may be NULL except where with_pose3d needs keypoint_coord3d).  Enqueue-only, allocates
 * nothing, capturable into a CUDA graph.  A track step adds fewer kernels to h3d_launch_count than a detect step by exactly
 * HandSegNet and the mask post-processing.  H3D_EINVAL before anything is enqueued unless 1 <= H, W <= H3D_PIPELINE_MAX_SIDE, B >= 1,
 * state is 8-byte aligned, margin is finite and >= 0.25, and min_score is finite or NaN (NaN = no score test). */
H3D_API int h3d_track_step(h3d_ctx* ctx, const float* image, const float* hand_side, int B, int H, int W, int with_pose3d, int detect,
                           float margin, float min_score, void* state, float* image_crop, float* scale_crop, float* center,
                           float* keypoints_scoremap, float* keypoint_coord3d, int32_t* keypoints_uv, void* stream);
/* A track step that re-detects only the slots that need it.  In stream order:
 *   1. select: slot b is selected when the state's lost[b] != 0 (written by the previous step's update) or force[b] != 0 (force: optional
 *      device int32 [B], NULL = none).  A fresh state (lost = 1 everywhere) selects every slot.  The count and the selected slots, in
 *      ascending order, live in context-owned device memory, not in the workspace;
 *   2. HandSegNet and the mask post-processing on the selected slots only: a device-counted batch whose first layer reads slot slots[i]
 *      of `image` in place, every kernel bounded by the count on the device.  A slot's result has the same bits as in a detect step;
 *   3. merge: a selected slot takes the crop its mask gives, every other slot its state's crop;
 *   4. the crop, PoseNet2D, key-points and lifting on every slot, then the update, as in h3d_track_step.
 * So every output of a selected slot equals h3d_track_step with detect != 0, and of any other slot detect == 0, bit for bit.
 * detected (optional, device int32 [B]) receives 1 for the selected slots, 0 for the others.  The host never reads the selection, so a
 * slot lost at step t is re-detected at step t + 1.  With no slot selected the counted kernels exit at once.  The first call for a
 * (B, H, W) builds the counted plan (outside any graph capture); after that the entry only enqueues, allocates nothing and is
 * capturable.  Argument rules as h3d_track_step's; a refused call enqueues nothing. */
H3D_API int h3d_track_step_slots(h3d_ctx* ctx, const float* image, const float* hand_side, int B, int H, int W, int with_pose3d,
                                 float margin, float min_score, void* state, const int32_t* force, int32_t* detected, float* image_crop,
                                 float* scale_crop, float* center, float* keypoints_scoremap, float* keypoint_coord3d,
                                 int32_t* keypoints_uv, void* stream);
/* The update alone (the operator form of h3d_track_step's last kernel): scoremap32 [B,32,32,21] (the last PoseNet2D stage),
 * keypoints_uv [B,21,2] int32, center [B,2] and scale_crop [B] of the crop they were found in -> state.  Same argument rules. */
H3D_API int h3d_track_update(h3d_ctx* ctx, const float* scoremap32, const int32_t* keypoints_uv, const float* center,
                             const float* scale_crop, int B, float margin, float min_score, void* state, void* stream);

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
/* One network layer as the stage entries build it, with its raw output planes (for tests of the layer paths the stage plans use).
 * x fp32 [B,H,W,Cx]; host_w_hwio [k,k,Cin,Cout] and host_bias [Cout] are HOST pointers.  precision: a tensor-core mode.
 * route 0: the wgmma layer.  x is split on the device into the precision's planes with Cin_total = Cx (Cx % 16 == 0); the layer reads
 *   channels [0, Cin_pad), Cin_pad = align_up(Cin, 64) <= Cx.  host_perm (NULL = identity) is host int32 [Cin_pad]: packed input
 *   channel j takes weight row host_perm[j], -1 = a zero row (PoseNet2D's conv6_1 / conv7_1 read the concat planes this way).
 *   pool: 0, 1 = fused 2x2 max-pool, 2 = stride 2; outputs are [B,H/2,W/2,.] when pool != 0.
 * route 1: the CUDA-core layer; a 3x3, 3 -> 64 layer runs the first-layer kernels (the tensor-core one when only planes are
 *   requested, the FFMA one with yf, with the c3_ffma switch, or in fp16_f8c).  pool must be 0 and host_perm NULL.
 * Outputs (each optional, at least one): planes [B,Ho,Wo,Cy_total] at channel offset cy_off, y_hi (uint16) always, y_lo (uint16) in
 * bf16x3 / fp16x3, y_l8 and y_h8 (uint8) in fp16_f8c; plane pointers the precision does not use are never written.  Route 0 writes
 * Cout_pad = align_up(Cout, 64) plane channels, the padding ones as zeros; yf fp32 [B,Ho,Wo,Cyf_total] gets Cout channels at cyf_off.
 * Descriptor errors (alignment of the offsets, pool with Cout % 32 != 0 or odd H / W, ...) return H3D_EINVAL.  Like h3d_conv2d_tc, the
 * call uploads the host weights and frees them afterwards (the free waits for the kernel); the input planes live in the operator
 * scratch. */
H3D_API int h3d_conv2d_layer_planes(h3d_ctx* ctx, const float* x, int B, int H, int W, int Cx, const float* host_w_hwio,
                                    const float* host_bias, int ksize, int Cin, int Cout, const int32_t* host_perm, int pool, int leaky,
                                    int precision, int route, void* y_hi, void* y_lo, void* y_l8, void* y_h8, int Cy_total, int cy_off,
                                    float* yf, int Cyf_total, int cyf_off, void* stream);
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
/* Which tile the tensor-core convolution runs a layer on, from the library's own choosers (host only: no context, no device, nothing
 * is launched; without a device the SM count is taken as 132).  For tests and tools that must know which kernel geometry a shape
 * exercises.  out[4] = TW, TH, TB, BN: a pixel tile of TW x TH pixels of TB images (TW * TH * TB = 128 rows) and the N tile (64 or 128
 * output channels), for x [B,H,W,.] -> Cout channels with pool as in h3d_conv2d_layer_planes (stride 2 of the operator entries is
 * pool = 2), under the current "tc_bn" tuning.  The data gradient of h3d_conv2d_tc_backward is this geometry with Cout = the layer's
 * Cin and pool = 0. */
H3D_API int h3d_conv2d_tc_geometry(int B, int H, int W, int Cout, int pool, int precision, int* out);
/* The weight-gradient kernel's geometry for h3d_conv2d_tc_backward on x [B,H,W,Cin] (H, W of the layer's input at either stride):
 * out[6] = TW, TH, TB (a 64-pixel box), BN (64 or 128 input channels per tile), num_tiles (ksize^2 x Cout tiles x Cin tiles) and
 * splits (CTAs that share one tile's pixel blocks). */
H3D_API int h3d_conv2d_wgrad_geometry(int B, int H, int W, int ksize, int Cin, int Cout, int* out);
/* The kernels of the fp32 CUDA-core convolution (h3d_conv2d_f32, and route 1 of h3d_conv2d_layer_planes): */
#define H3D_DIRECT_C3_TC 0      /* first layer (3x3, 3 -> 64, stride 1) on the tensor cores, planes only */
#define H3D_DIRECT_C3_FFMA 1    /* first layer on the register-tiled FFMA kernel */
#define H3D_DIRECT_VEC 2        /* generic kernel, float4 gathers (Cin % 16 == 0, 16-byte aligned input channels) */
#define H3D_DIRECT_SCALAR 3     /* generic kernel, scalar gathers */
/* Split-K scratch (floats) the library's entries give the generic kernel. */
#define H3D_CONV_SPLITK_SCRATCH_FLOATS (600LL * 64 * 64)
/* Which kernel, grid and split of K the CUDA-core convolution runs a layer on, from the launcher's own choosers (host only, like
 * h3d_conv2d_tc_geometry).  The layer reads channels [cin_off, cin_off + Cin) of x [B,H,W,Cin_total]; x_aligned says whether those
 * channels start 16 bytes aligned.  It writes fp32 output when yf != 0 (Cout channels at cout_off of Cout_total) and/or the planes of
 * precision `planes` (a tensor-core mode, H3D_PREC_FP32_FFMA = none; Cout channels at cs_off of Cs_total).  splitk_scratch_floats is
 * the split-K scratch offered (0 = none; h3d_conv2d_f32 offers H3D_CONV_SPLITK_SCRATCH_FLOATS when B ceil(H/s) ceil(W/s) <= 64 x 295,
 * the stage entries always), under the current "c3_ffma" tuning.  out[6] = kernel (H3D_DIRECT_*), grid x, y, z, ksplit (2 launches when
 * > 1: the partial sums, then their fixed-order reduction) and k_per_split (reduction rows per blockIdx.z).  The first-layer kernels
 * do not split K (k_per_split = 27); the grid of H3D_DIRECT_C3_TC depends on the device's SM count and is reported as 0 x 0 x 0. */
H3D_API int h3d_conv2d_f32_geometry(int B, int H, int W, int Cin, int Cin_total, int cin_off, int Cout, int Cout_total, int cout_off,
                                    int yf, int planes, int Cs_total, int cs_off, int ksize, int stride, int x_aligned,
                                    int64_t splitk_scratch_floats, int* out);
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
/* Its split of K, from the launcher's own chooser (host only): out[5] = ksplit, k_per_split, grid x (64-output tiles), y (= ksplit),
 * z (32-row batch tiles).  Every call is two launches: the partial sums, then their fixed-order reduction. */
H3D_API int h3d_fully_connected_f32_geometry(int B, int in_features, int out_features, int* out);
/* tf.image.resize_images bilinear, align_corners=False, TF1 legacy (nets/...:97,128,166). */
H3D_API int h3d_resize_bilinear_tf1(h3d_ctx* ctx, const float* x, float* y, int B, int H, int W, int C,
                            int out_h, int out_w, void* stream);
/* tf.nn.avg_pool 8x8/8 (nets/PosePriorNetwork.py:61). */
H3D_API int h3d_avgpool8(h3d_ctx* ctx, const float* x, float* y, int B, int H, int W, int C, void* stream);
/* single_obj_scoremap + calc_center_bb + crop-scale glue (utils/general.py:233-328,
 * nets/ColorHandPose3DNetwork.py:83-85).  logits [B,H,W,2] -> hand_mask [B,H,W] uint8 (optional),
 * max_loc [B,2] int32 (optional, find_max_location), center [B,2], crop_size [B,1] (raw, optional),
 * scale_crop [B,1].  1 <= H, W <= H3D_PIPELINE_MAX_SIDE and B <= 65535 (else H3D_EINVAL before anything is enqueued),
 * W % 32 == 0 not required.  Up to 512 a side one CTA grows the mask; larger maps are split into row bands over a thread-block
 * cluster, with the same result. */
H3D_API int h3d_seg_postprocess(h3d_ctx* ctx, const float* logits, int B, int H, int W, uint8_t* hand_mask,
                        int32_t* max_loc, float* center, float* crop_size, float* scale_crop, void* stream);
/* calc_center_bb (utils/general.py:271-328) on an arbitrary mask [B,H,W] fp32 (pixels with int(mask) == 1 count):
 * center [B,2] (row, col), bb [B,2,2] = [[x_min, x_max], [y_min, y_max]] (optional), crop_size [B,1] (optional); an empty mask
 * gives center (160, 160), crop_size 100, bb (+inf, -inf) as the reference's tf.cond fall-backs do. */
H3D_API int h3d_calc_center_bb(h3d_ctx* ctx, const float* mask, int B, int H, int W, float* center, float* bb, float* crop_size,
                               void* stream);
/* crop_image_from_xy (utils/general.py:163-196) incl. tf.image.crop_and_resize bilinear/extrapolation 0.  1 <= B <= 65535,
 * crop_size^2 <= 2^31 - 1. */
H3D_API int h3d_crop_image_from_xy(h3d_ctx* ctx, const float* image, const float* center, const float* scale,
                           float* image_crop, int B, int H, int W, int C, int crop_size, void* stream);
/* detect_keypoints (utils/general.py:331-344), batched: scoremaps [B,H,W,C] -> [B,C,2] int32 (row,col) of np.argmax per channel:
 * the first occurrence of the maximum in row-major order, where -0.0 ties +0.0 and every NaN (either sign) ranks above +inf, so the
 * first NaN wins.  1 <= C <= 256, 1 <= B <= 65535, H W <= 2^31 - 1. */
H3D_API int h3d_detect_keypoints(h3d_ctx* ctx, const float* scoremaps, int B, int H, int W, int C,
                         int32_t* keypoints_uv, void* stream);
/* tf.image.resize_images (nets/ColorHandPose3DNetwork.py:96-97) fused with detect_keypoints: 21-channel score maps [B,H,W,21] ->
 * scoremaps_up [B,out_h,out_w,21] and keypoints_uv [B,21,2] int32 (row, col) of the up-sampled maps in one pass, with the arg-max
 * rules of h3d_detect_keypoints.  1 <= B <= 65535, out_h out_w <= 2^31 - 1. */
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
/* ---- Training-mode augmentation of the RHD reader (data/BinaryDbReader.py:160-401 with its seven flags) ----
 * Every random value is a pure function of (seed, serial, value id, attempt): serial is the sample's position in the ENQUEUE stream
 * (record = serial mod records in the file), so a sample's augmentation depends neither on the batch size nor on the shuffle.
 * Generator: Philox4x64-10 (Salmon et al., SC'11; numpy.random.Philox is the same function), key = (seed, H3D_AUG_STREAM_ITEMS),
 * counter = (serial, value id, attempt, 0), four 64-bit words per call.  The value id is the parameter's index in the layout below.
 *   uniform fp32 in [0, 1)   = (w0 >> 40) * 2^-24 (exact), then TF's random_uniform affine step u * (max - min) + min in fp32;
 *   truncated normal         = Box-Muller in fp64 on (w0, w1) of attempt a = 0, 1, ...: z0 = r cos(2 pi u2), z1 = r sin(2 pi u2),
 *                              u1 = ((w0 >> 11) + 1) 2^-53, u2 = (w1 >> 11) 2^-53; the first of z0, z1, z0', z1', ... with
 *                              |z| <= 2 is kept (rounded to fp32), then TF's z * stddev + 0 in fp32; after H3D_AUG_MAX_ATTEMPTS
 *                              attempts without one (probability ~1e-43) z = 0;
 *   window offset in [0, 64] = w0 mod 65;  keep bit = floor(0.8f + u) in fp32 (TF 1.3 dropout, keep_prob 0.8).
 * The shuffle queue's dequeue order comes from a separate key (seed, H3D_AUG_STREAM_SHUFFLE); h3d_reader_next_serials runs it on the
 * device, and the Python reader's host queue draws the same words. */
#define H3D_AUG_STREAM_ITEMS 0
#define H3D_AUG_STREAM_SHUFFLE 1
#define H3D_AUG_MAX_ATTEMPTS 16
/* flags */
#define H3D_AUG_COORD_UV_NOISE 1     /* truncated normal, sigma 2.5 px, on the 42 palm-substituted keypoint_uv (:160-164) */
#define H3D_AUG_CROP_CENTER_NOISE 2  /* truncated normal, sigma 20 px, on the crop centre before the crop size (:277-279) */
#define H3D_AUG_CROP_SCALE_NOISE 4   /* U[1, 1.2) factor on the clamped crop scale (:281-283, 307) */
#define H3D_AUG_CROP_OFFSET_NOISE 8  /* truncated normal, sigma 10 px, on the crop centre after the crop size (:310-312) */
#define H3D_AUG_HUE 16               /* tf.image.random_hue(image, 0.1) on image / 255 - 0.5 (:183-184) */
#define H3D_AUG_RANDOM_CROP 32       /* one 256 x 256 window of image, hand_parts, hand_mask, offsets in [0, 64] (:382-392) */
#define H3D_AUG_SCOREMAP_DROPOUT 64  /* per key-point keep bits, keep 0.8, then * 0.8 (:362-365) */
/* per-sample parameter layout: params [B, H3D_AUG_PARAMS] fp32, FINAL values (px, factors, offsets, bits), not standard draws */
#define H3D_AUG_UV_NOISE 0           /* [42][2] (u, v) px */
#define H3D_AUG_CENTER_NOISE 84      /* [2] (row, col) px */
#define H3D_AUG_SCALE 86             /* [1] factor in [1, 1.2) */
#define H3D_AUG_OFFSET_NOISE 87      /* [2] (row, col) px */
#define H3D_AUG_HUE_DELTA 89         /* [1] in [-0.1, 0.1) */
#define H3D_AUG_WINDOW 90            /* [2] (row, col) offsets, integers in [0, 64] stored as floats */
#define H3D_AUG_KEEP 92              /* [21] 0 or 1 */
#define H3D_AUG_USED 113
#define H3D_AUG_PARAMS 128
/* serials [B] int64 (device) -> params [B, H3D_AUG_PARAMS]: the final value of every flag in `flags`; a flag that is off gets its
 * neutral value (0 px, factor 1, delta 0, offset 0, keep 1) and unused slots are 0. */
H3D_API int h3d_reader_aug_params(h3d_ctx* ctx, const int64_t* serials, int B, uint64_t seed, int flags, float* params, void* stream);
/* ---- Device-resident reading: the record stream and the record gather, with no host in the loop (capturable) ----
 * Queue state: H3D_READER_STATE_WORDS int64 words of DEVICE memory owned by the caller:
 *   [H3D_READER_STATE_COUNT] dequeues so far, [H3D_READER_STATE_NEXT] next stream position to enqueue,
 *   [H3D_READER_STATE_SLOTS + k] stream position held by queue slot k (shuffle only).
 * A fresh queue is count 0 and, with shuffle, next 100 and slot k = k (the first 100 stream positions); in order, next 0. */
#define H3D_READER_QUEUE_CAPACITY 100
#define H3D_READER_STATE_COUNT 0
#define H3D_READER_STATE_NEXT 1
#define H3D_READER_STATE_SLOTS 2
#define H3D_READER_STATE_WORDS 102
#define H3D_READER_MAX_GATHER 4096
/* The next B serials (stream positions) of the reader's queue -> serials [B] int64 (device); advances state.  Without shuffle they are
 * next, next + 1, ...  With shuffle (shuffle_batch_join(capacity=100, min_after_dequeue=50) in its steady state), dequeue n takes slot
 * k = w_n mod 100 and refills it with next++, where w_n is word n of Philox4x64-10 keyed (seed, H3D_AUG_STREAM_SHUFFLE) in
 * numpy.random.Philox.random_raw order: word (n mod 4) of the block at counter (n / 4 + 1, 0, 0, 0) (numpy increments the counter before
 * it fills its 4-word buffer).  The stream depends on the seed and the dequeue count only, not on how it is cut into batches.
 * count < 2^63.  One CTA; enqueue-only. */
H3D_API int h3d_reader_next_serials(h3d_ctx* ctx, int64_t* state, int B, uint64_t seed, int shuffle, int64_t* serials, void* stream);
/* h3d_decode_records of records gathered from a resident file: file = n_records whole records of `dataset` back to back (device),
 * serials [B] int64 (device, >= 0); sample b is record serials[b] mod n_records, decoded exactly as h3d_decode_records decodes it.
 * B <= H3D_READER_MAX_GATHER; outputs as h3d_decode_records. */
H3D_API int h3d_decode_records_gather(h3d_ctx* ctx, int dataset, const uint8_t* file, int64_t n_records, const int64_t* serials, int B,
                                      int step, float* header, float* image, uint8_t* mask, uint8_t* visibility, void* stream);

/* ---- camera frames (run.py:57-59: image_raw = scipy.misc.imresize(image_raw, (240, 320)); image_raw.astype('float') / 255.0 - 0.5)
 * frames [B,H,W,3] uint8 RGB, contiguous (device) -> out [B,out_h,out_w,3]: with normalize = 0 uint8, exactly scipy.misc.imresize(frame,
 * (out_h, out_w)) with interp='bilinear', i.e. Pillow's Image.resize((out_w, out_h), BILINEAR) (8-bit fixed point, 22 fractional bits,
 * horizontal pass into uint8 first, no pass on an axis that keeps its size); with normalize = 1 float32, run.py's network input
 * float32(float64(u) / 255.0 - 0.5) of that uint8 result.  1 <= H, W <= H3D_FRAME_MAX_SIDE and 1 <= out_h, out_w <= H3D_FRAME_MAX_OUT,
 * anything else is H3D_EINVAL.  The first call with a new (H, W, out_h, out_w) builds its coefficients on the host and uploads them on
 * `stream`; such a call is refused while `stream` is being captured.  Later calls only enqueue one kernel (capturable); a context keeps
 * every plan until h3d_destroy. */
#define H3D_FRAME_MAX_SIDE 4096
#define H3D_FRAME_MAX_OUT 512
H3D_API int h3d_resize_frames(h3d_ctx* ctx, const uint8_t* frames, int B, int H, int W, int out_h, int out_w, int normalize, void* out,
                              void* stream);
/* Pixel formats of camera frames (B frames back to back, contiguous, uint8; H x W is the picture):
 *   H3D_PIXEL_RGB   [B,H,W,3] packed R G B (h3d_resize_frames' input)            1 <= H, W <= H3D_FRAME_MAX_SIDE
 *   H3D_PIXEL_BGR   [B,H,W,3] packed B G R (OpenCV's VideoCapture)               1 <= H, W <= H3D_FRAME_MAX_SIDE
 *   H3D_PIXEL_NV12  [B,H*3/2,W]: H rows of Y, then H/2 rows of interleaved U V   H, W even, 2..H3D_FRAME_MAX_SIDE
 *   H3D_PIXEL_I420  [B,H*3/2,W] as flat bytes: H*W of Y, then (H/2)(W/2) of U, then (H/2)(W/2) of V (ffmpeg's yuv420p)
 *                                                                                H, W even, 2..H3D_FRAME_MAX_SIDE
 *   H3D_PIXEL_YUYV  [B,H,W,2]: Y0 U Y1 V per pixel pair (YUY2, ffmpeg's yuyv422) 1 <= H <= H3D_FRAME_MAX_SIDE, W even, 2..H3D_FRAME_MAX_SIDE
 * The YUV formats are converted to RGB as OpenCV's cvtColor COLOR_YUV2RGB_NV12 / _I420 / _YUYV converts them: BT.601 limited range in
 * 20-bit fixed point, chroma replicated (not interpolated).  Pixel (y, x) takes its luma Y and the chroma (U, V) at (y/2, x/2) (4:2:0) or
 * (y, x/2) (YUYV); c = max(Y - 16, 0) * 1220542 + (1 << 19), u = U - 128, v = V - 128, and with an arithmetic shift, clipped to 0..255:
 *   R = (c + 1673527 v) >> 20,   G = (c - 852492 v - 409993 u) >> 20,   B = (c + 2116026 u) >> 20.
 * This is not ffmpeg/swscale's rgb24 conversion, which rounds and interpolates chroma differently. */
#define H3D_PIXEL_RGB 0
#define H3D_PIXEL_BGR 1
#define H3D_PIXEL_NV12 2
#define H3D_PIXEL_I420 3
#define H3D_PIXEL_YUYV 4
/* h3d_resize_frames of frames in `format` (H3D_PIXEL_*): out is Pillow's BILINEAR resize (and with normalize = 1 run.py's
 * normalisation) of the frames converted to RGB by the rule above, bit for bit; BGR is the resize of the channel-reversed frame.  With
 * H3D_PIXEL_RGB it is h3d_resize_frames.  The conversion is fused into the resize kernel (one instance per format), so nothing but `out`
 * is written.  Sizes per the table above and 1 <= out_h, out_w <= H3D_FRAME_MAX_OUT, anything else (or an unknown format) is H3D_EINVAL
 * before anything is enqueued.  Plans are kept per (format, H, W, out_h, out_w) and built as h3d_resize_frames builds them. */
H3D_API int h3d_resize_frames_fmt(h3d_ctx* ctx, const uint8_t* frames, int format, int B, int H, int W, int out_h, int out_w, int normalize,
                                  void* out, void* stream);
/* frames in `format` -> out_rgb [B,H,W,3] uint8 RGB at full size, by the rule above (RGB: a copy; BGR: the channels reversed).  Sizes
 * per the table above, else H3D_EINVAL before anything is enqueued.  Enqueues one kernel and allocates nothing (capturable). */
H3D_API int h3d_convert_frames(h3d_ctx* ctx, const uint8_t* frames, int format, int B, int H, int W, uint8_t* out_rgb, void* stream);
/* Camera rigs (a size and a pixel format per batch slot): include/hand3d_b200_rig.h. */
#include "hand3d_b200_rig.h"
/* tf.image.random_hue (TF 1.3 adjust_hue, non-fused: rgb_to_hsv, h = mod(h + (delta + 1), 1), hsv_to_rgb, in the functors' fp32 order)
 * and / or the random_crop window, in one pass.  image [B,H,W,3] fp32, hand_parts [B,H,W] u8, params as above (delta at
 * H3D_AUG_HUE_DELTA when flags has H3D_AUG_HUE, window at H3D_AUG_WINDOW when flags has H3D_AUG_RANDOM_CROP) -> out_image [B,h,w,3]
 * and, with the window, out_parts [B,h,w] int32 and out_mask [B,h,w,2] int32 (background, hand) (each may be NULL); (h, w) = (window,
 * window) with H3D_AUG_RANDOM_CROP, else (H, W). */
H3D_API int h3d_augment_image(h3d_ctx* ctx, const float* image, const uint8_t* hand_parts, const float* params, int B, int H, int W,
                              int flags, int window, float* out_image, int32_t* out_parts, int32_t* out_mask, void* stream);
/* h3d_rhd_reader_items with the coordinate and crop noises of `flags` (H3D_AUG_COORD_UV_NOISE, _CROP_CENTER_NOISE, _CROP_SCALE_NOISE,
 * _CROP_OFFSET_NOISE) read from params [B, H3D_AUG_PARAMS]; params may be NULL when flags is 0, which computes exactly what
 * h3d_rhd_reader_items computes.  keypoint_uv [B,42,2] (may be NULL) is the reader's keypoint_uv item: palm-substituted when
 * use_wrist_coord == 0, noisy with H3D_AUG_COORD_UV_NOISE.  crop_center is the final centre (both noises applied). */
H3D_API int h3d_rhd_reader_items_aug(h3d_ctx* ctx, const float* header, const uint8_t* hand_parts, const uint8_t* visibility, int B,
                                     int use_wrist_coord, int hand_crop, int crop_size, const float* params, int flags,
                                     float* keypoint_uv, float* keypoint_xyz21, float* keypoint_uv21, uint8_t* keypoint_vis21,
                                     float* hand_side, float* keypoint_scale, float* keypoint_xyz21_normed, float* crop_center,
                                     float* crop_scale, float* cam_mat, void* stream);
/* h3d_gaussian_scoremap followed by TF 1.3 dropout with one keep bit per (sample, key-point) and the reader's rescale:
 * out = ((map / keep_prob) * keep[b * keep_stride + n]) * keep_prob, each step rounded in fp32. */
H3D_API int h3d_gaussian_scoremap_dropout(h3d_ctx* ctx, const float* coords_hw, const uint8_t* valid, const float* keep, int keep_stride,
                                          float keep_prob, int B, int N, int H, int W, float sigma, float* scoremap, void* stream);
/* canonical_trafo (+ flip_right_hand, + the tf.matrix_inverse the readers apply) (utils/canonical_trafo.py:97-162,
 * data/BinaryDbReader.py:247-252): coords_xyz [B,21,3] -> coords_can [B,21,3] (z mirrored where cond_right[b] != 0; cond_right may be
 * NULL), rot_mat [B,3,3] (total rotation), rot_mat_inv [B,3,3]; each output may be NULL. */
H3D_API int h3d_canonical_trafo(h3d_ctx* ctx, const float* coords_xyz, const uint8_t* cond_right, int B, float* coords_can, float* rot_mat,
                                float* rot_mat_inv, void* stream);
/* EvalUtil.feed (utils/general.py:531-549), batched on device: gt / pred [n, D] (D = 2 or 3), vis [n] u8 ->
 * dist [n] = ||gt - pred||_2, or -1 where the key-point is not visible. */
H3D_API int h3d_eval_keypoint_dist(h3d_ctx* ctx, const float* gt, const uint8_t* vis, const float* pred, int n, int D, float* dist,
                                   void* stream);
/* ---- EvalUtil on the device (utils/general.py:522-611): a store of per-key-point distance lists and its measures ----
 * A store is caller-owned DEVICE memory of h3d_eval_store_bytes(K, num_samples, dtype) bytes:
 *   int64 header [H3D_EVAL_HEADER_WORDS]: [H3D_EVAL_KEPT] samples kept, [H3D_EVAL_DROPPED] rows dropped, [H3D_EVAL_TICKET] scratch
 *   of h3d_eval_feed (0 between calls), [H3D_EVAL_COUNT + k] distances held for key-point k;
 *   then K x num_samples distance slots of the store's dtype: key-point k's list at slot k * num_samples.
 * Zeroing the header (a memset of H3D_EVAL_HEADER_WORDS * 8 bytes) resets the store.  dtype is H3D_EVAL_FLOAT32 or H3D_EVAL_FLOAT64;
 * 1 <= K <= H3D_EVAL_MAX_KP, 1 <= num_samples <= H3D_EVAL_MAX_SAMPLES, 1 <= D <= H3D_EVAL_MAX_DIM, 1 <= T <= H3D_EVAL_MAX_THRESHOLDS;
 * anything else is H3D_EINVAL. */
#define H3D_EVAL_FLOAT32 0
#define H3D_EVAL_FLOAT64 1
#define H3D_EVAL_KEPT 0
#define H3D_EVAL_DROPPED 1
#define H3D_EVAL_TICKET 2
#define H3D_EVAL_COUNT 8
#define H3D_EVAL_HEADER_WORDS 72
#define H3D_EVAL_MAX_KP 64
#define H3D_EVAL_MAX_DIM 4
#define H3D_EVAL_MAX_SAMPLES 16777216
#define H3D_EVAL_MAX_THRESHOLDS 4096
/* h3d_eval_stats output: int64 [K][H3D_EVAL_STAT_COUNTS + T]; the mean and median are float64 bit patterns (exact for float32). */
#define H3D_EVAL_STAT_N 0
#define H3D_EVAL_STAT_MEAN 1
#define H3D_EVAL_STAT_MEDIAN 2
#define H3D_EVAL_STAT_COUNTS 3
/* Bytes of a store, or H3D_EINVAL (< 0) outside the limits. */
H3D_API int64_t h3d_eval_store_bytes(int K, int num_samples, int dtype);
/* EvalUtil.feed of n samples: gt / pred [n, K, D] and vis [n, K] u8 (nonzero = visible), contiguous, in the store's dtype (device).
 * Key-point k of sample r gets np.sqrt(np.sum(np.square(gt - pred), axis=1)) in that dtype (as h3d_eval_keypoint_dist, in float64 too),
 * appended to its list when visible: lists grow in feed order, then sample order, as the reference's per-sample loop appends.  Samples
 * past the store's num_samples are not stored but counted as dropped.  No atomics decide positions: the store is deterministic.
 * One kernel, enqueue-only and capturable. */
H3D_API int h3d_eval_feed(h3d_ctx* ctx, void* store, int K, int num_samples, int dtype, const void* gt, const uint8_t* vis,
                          const void* pred, int n, int D, void* stream);
/* The measures of every key-point k with n_k > 0 (one kernel): n_k, np.mean of its list (numpy 2.x pairwise summation, then / n_k, in
 * the store's dtype), np.median (the middle order statistic, or (a + b) / 2 in the store's dtype; NaN if the list holds NaN) and
 * counts[t] = #{d : float64(d) <= thresholds[t]} for thresholds [T] float64 (device).  A key-point with no data gets a row of zeros. */
H3D_API int h3d_eval_stats(h3d_ctx* ctx, const void* store, int K, int num_samples, int dtype, const double* thresholds, int T,
                           int64_t* out, void* stream);
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
 * sqrt(mean (pred - target)^2), which the backward reuses.  fp32 with separate multiply and add.  Any B >= 1 is accepted (no
 * per-image grid limit). */
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

/* ---- Training of the lifting stage (training_lifting.py); the same conventions as the section above ---- */

/* Adjoint of h3d_rotate_canonical (out = flip_z(can) R, R = Rodrigues(uxyz), the flip where argmax(hand_side) == 1): can [B,21,3],
 * uxyz [B,3], hand_side [B,2], and the incoming gradients d_out [B,21,3] and d_R [B,3,3], either of which may be NULL (= 0) ->
 * d_can [B,21,3], d_uxyz [B,3].  R is recomputed with the forward's own fp32 operations; the sum over the 21 key-points for dR runs
 * in ascending order. */
H3D_API int h3d_rotate_canonical_backward(h3d_ctx* ctx, const float* coord_can, const float* uxyz, const float* hand_side,
                                          const float* d_out, const float* d_rot_mat, int B, float* d_can, float* d_uxyz, void* stream);
/* Adjoint of h3d_bone_rel_trafo_inv: coords_rel [B,21,3] (the forward's input), d_xyz [B,21,3] -> d_rel [B,21,3]. */
H3D_API int h3d_bone_rel_trafo_inv_backward(h3d_ctx* ctx, const float* coords_rel, const float* d_xyz, float* d_rel, int B, void* stream);
/* bone_rel_trafo (utils/relative_trafo.py:184-240): xyz [B,21,3] -> (length, angle_x, angle_y) [B,21,3] per bone, with the reference's
 * own atan2 (atan(y / (x + 1e-8)) plus quadrant corrections).  The 'local' variant's training target. */
H3D_API int h3d_bone_rel_trafo(h3d_ctx* ctx, const float* coords_xyz, float* coords_rel, int B, void* stream);
/* reduce_mean(square(pred - target)) over n elements -> loss (device scalar). */
H3D_API int h3d_mse_loss_forward(h3d_ctx* ctx, const float* pred, const float* target, int64_t n, float* loss, void* stream);
/* Its gradient: dpred [n] = (grad_loss / n) (2 (pred - target)). */
H3D_API int h3d_mse_loss_backward(h3d_ctx* ctx, const float* pred, const float* target, const float* grad_loss, int64_t n, float* dpred,
                                  void* stream);

/* ---- Dropout of the lifting stage (ops.dropout, utils/general.py:139-148: evaluation = False) ----
 * TF 1.3's tf.nn.dropout in fp32: keep bit k = floor(keep_prob + u), y = (x / keep_prob) * k (a rounded division, then a rounded
 * multiply), and the gradient dx = (dy * k) / keep_prob (TF's Mul gradient, then its RealDiv gradient).  keep_prob == 1 keeps every
 * element and returns x bit for bit.
 * Draws are the project's own, not TF's streams: Philox4x64-10 (as for the reader) keyed (seed, H3D_DROPOUT_STREAM), counter
 * (draw, layer, row, col / 4); element (row, col) takes word col mod 4 and u = (w >> 40) 2^-24 (exact in fp32).
 * Layers: H3D_DROPOUT_LAYER_FC_REL0 / _FC_REL1 (PosePrior, keep 0.8, nets/PosePriorNetwork.py:113-114), _FC_VP0 / _FC_VP1 (ViewpointNet,
 * keep 0.75, :151-154); NetworkOps.dropout uses H3D_DROPOUT_LAYER_OP.  row is the sample's index in the batch.
 * One generator per context: a seed and the int64 `draw` counter in context-owned device memory.  Every dropout kernel reads draw on
 * the device, and the advance kernel adds 1 to it there, so a captured graph draws fresh masks on every replay and the host never reads
 * the counter. */
#define H3D_DROPOUT_STREAM 2
#define H3D_DROPOUT_LAYER_FC_REL0 0
#define H3D_DROPOUT_LAYER_FC_REL1 1
#define H3D_DROPOUT_LAYER_FC_VP0 2
#define H3D_DROPOUT_LAYER_FC_VP1 3
#define H3D_DROPOUT_LAYER_OP 4
/* enabled != 0: dropout on with `seed`; draw is set to 0 on the first enabling and whenever the seed changes (a synchronous write: not
 * while a stream is being captured).  enabled == 0: off (the default); seed and draw are kept, so enabling again with the same seed
 * continues the stream.  While it is on, every lifting computation of the context (h3d_lifting_forward, h3d_pipeline_forward with
 * with_pose3d, h3d_track_step, h3d_track_step_slots) applies the four layers above after the hidden FC layers, layer by layer, and then
 * adds 1 to draw: one forward is one draw.  Off, they compute exactly what they compute without this entry.  The context keeps one plan
 * for each setting, so switching between calls rebuilds nothing. */
H3D_API int h3d_set_dropout(h3d_ctx* ctx, int enabled, uint64_t seed);
/* *draw = the device address of the counter (int64), so that a caller can save and restore the stream. */
H3D_API int h3d_dropout_draw(h3d_ctx* ctx, int64_t** draw);
/* x [rows, cols] fp32 (device) -> y [rows, cols] fp32 (may be x) and keep [rows, cols] uint8 (0 / 1; may be NULL) at the current draw.
 * Does not advance the draw.  0 < keep_prob <= 1, rows, cols >= 1, layer >= 0 and dropout enabled, else H3D_EINVAL with nothing
 * enqueued.  These entries only enqueue: no allocation, no synchronisation (capturable). */
H3D_API int h3d_dropout_forward(h3d_ctx* ctx, const float* x, int rows, int cols, float keep_prob, int layer, float* y, uint8_t* keep,
                                void* stream);
/* The same, also writing the 16-bit planes a tensor-core FC layer reads: hi = h16(y), lo = h16(y - hi) (lo may be NULL), [rows, stride]
 * with stride >= cols and zeros in the columns [cols, stride); h16 is bf16 (half = 0) or fp16 (half = 1), round to nearest even. */
H3D_API int h3d_dropout_forward_planes(h3d_ctx* ctx, const float* x, int rows, int cols, float keep_prob, int layer, float* y, uint8_t* keep,
                                       int half, int stride, uint16_t* hi, uint16_t* lo, void* stream);
/* dy, keep [rows, cols] -> dx = (dy * keep) / keep_prob (may be dy); the same argument rules. */
H3D_API int h3d_dropout_backward(h3d_ctx* ctx, const float* dy, const uint8_t* keep, int rows, int cols, float keep_prob, float* dx,
                                 void* stream);
/* Adds 1 to draw on the device (one kernel). */
H3D_API int h3d_dropout_advance(h3d_ctx* ctx, void* stream);

/* ---- drawing (utils/general.py:360-477, plot_hand / plot_hand_3d: the stick figures run.py shows)
 * Draws S anti-aliased segments into each of B uint8 RGB images [B,H,W,3] (device, contiguous), in place.  segments [B,S,4] float32
 * (device): (r0, c0, r1, c1) in pixels, pixel (y, x) centred at (y, x).  host_colors [S,3] float32 (HOST, 0..255) are copied into the
 * kernel's parameters, so a captured graph carries them.  valid [B] int32 (device) or NULL: an image with valid[b] == 0 is left alone.
 * The rule, in fp32 with no contraction: h = linewidth / 2 + 0.5; for each segment k in order whose four values are finite,
 * dy = r1 - r0, dx = c1 - c0, L2 = dy*dy + dx*dx, ry = y - r0, rx = x - c0, t = clamp(L2 > 0 ? (ry*dy + rx*dx) / L2 : 0, 0, 1)
 * (NaN -> 0), ey = ry - t*dy, ex = rx - t*dx, d = sqrt(ey*ey + ex*ex), a = clamp(h - d, 0, 1) (NaN -> 0); where a > 0 each channel
 * v = v + a * (C[k] - v), v starting as float(byte); the byte written is rint(v) clamped to 0..255.  Segment k reaches only the
 * pixels of its box min(r0, r1) - g <= y <= max(r0, r1) + g, min(c0, c1) - g <= x <= max(c0, c1) + g (g = h + 1, bounds in fp32);
 * outside it a = 0.  For end points within 2^14 px of the image the box changes nothing (d > h outside it); farther out x - c0 and
 * c1 - c0 can round alike, and the box keeps a long segment from drawing past its end.  A pixel no segment covers keeps its byte.
 * 1 <= H, W <= H3D_FRAME_MAX_SIDE, 1 <= S <= H3D_DRAW_MAX_SEGMENTS, 0 < linewidth <= H3D_DRAW_MAX_LINEWIDTH (finite), colours finite
 * in 0..255, no NULL but valid; anything else is H3D_EINVAL with nothing enqueued.  Enqueues one kernel whose grid
 * depends on (B, H, W) only; allocates nothing (capturable). */
#define H3D_DRAW_MAX_SEGMENTS 64
#define H3D_DRAW_MAX_LINEWIDTH 64
H3D_API int h3d_draw_segments(h3d_ctx* ctx, uint8_t* images, int B, int H, int W, const float* segments, int S, const float* host_colors,
                              const int32_t* valid, float linewidth, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* HAND3D_B200_H_ */

// Shared declarations for the hand3d_b200 CUDA sources (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <algorithm>
#include <cmath>
#include <string>

#include "../../include/hand3d_b200.h"

namespace h3d {

// ---------------------------------------------------------------- error plumbing
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);

#define H3D_CUDA(expr)                                                     \
    do {                                                                   \
        cudaError_t _e = (expr);                                           \
        if (_e != cudaSuccess) return h3d::cuda_fail(_e, #expr, __FILE__, __LINE__); \
    } while (0)

#define H3D_CHECK_LAUNCH() H3D_CUDA(cudaGetLastError())

#define H3D_REQUIRE(cond, ...)                 \
    do {                                       \
        if (!(cond)) {                         \
            h3d::set_error(__VA_ARGS__);       \
            return H3D_EINVAL;                 \
        }                                      \
    } while (0)

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline int64_t align_up(int64_t a, int64_t b) { return (a + b - 1) / b * b; }

constexpr float kNegSlope = 0.01f;  // utils/general.py:28

// Activation tensors on the tensor-core path are stored as two 16-bit planes (hi, lo) with
// x ~= hi + lo ("split" format); lo == nullptr in single-pass modes.
struct Split {
    uint16_t* hi = nullptr;   // bf16 / fp16 main plane
    uint16_t* lo = nullptr;   // 16-bit residual plane (3-pass modes)
    uint8_t* l8 = nullptr;    // e4m3 residual plane  (fp16_f8c mode, see split_fmt.cuh)
    uint8_t* h8 = nullptr;    // e4m3 coarse copy     (fp16_f8c mode)
};

enum class Half16 : int { BF16 = 0, FP16 = 1 };

// ---------------------------------------------------------------- Rodrigues rotation (nets/ColorHandPose3DNetwork.py:311-334)
// R[9] from the axis-angle vector (ux, uy, uz); separate multiply / add as the TF graph evaluates it.
__device__ __forceinline__ void rodrigues_rot_mat(float ux_b, float uy_b, float uz_b, float* R) {
    const float n2 = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(ux_b, ux_b), __fmul_rn(uy_b, uy_b)), __fmul_rn(uz_b, uz_b)), 1e-8f);
    const float theta = sqrtf(n2);
    const float st = sinf(theta), ct = cosf(theta);
    const float one_ct = __fsub_rn(1.0f, ct);
    const float nf = __fdiv_rn(1.0f, theta);
    const float ux = __fmul_rn(ux_b, nf), uy = __fmul_rn(uy_b, nf), uz = __fmul_rn(uz_b, nf);
#define H3D_M3(a, b_, c) __fmul_rn(__fmul_rn(a, b_), c)
    R[0] = __fadd_rn(ct, H3D_M3(ux, ux, one_ct));
    R[1] = __fsub_rn(H3D_M3(ux, uy, one_ct), __fmul_rn(uz, st));
    R[2] = __fadd_rn(H3D_M3(ux, uz, one_ct), __fmul_rn(uy, st));
    R[3] = __fadd_rn(H3D_M3(uy, ux, one_ct), __fmul_rn(uz, st));
    R[4] = __fadd_rn(ct, H3D_M3(uy, uy, one_ct));
    R[5] = __fsub_rn(H3D_M3(uy, uz, one_ct), __fmul_rn(ux, st));
    R[6] = __fsub_rn(H3D_M3(uz, ux, one_ct), __fmul_rn(uy, st));
    R[7] = __fadd_rn(H3D_M3(uz, uy, one_ct), __fmul_rn(ux, st));
    R[8] = __fadd_rn(ct, H3D_M3(uz, uz, one_ct));
#undef H3D_M3
}

// out[kp, j] = sum_i can[kp, i] R[i, j] with the right-hand mirror of z (nets/ColorHandPose3DNetwork.py:239-247,336-361)
__device__ __forceinline__ float rotate_canonical_point(const float* can_b, const float* R, int i, bool right) {
    const int kp = i / 3, j = i - kp * 3;
    const float cx = can_b[3 * kp], cy = can_b[3 * kp + 1];
    float cz = can_b[3 * kp + 2];
    if (right) cz = -cz;
    return cx * R[j] + cy * R[3 + j] + cz * R[6 + j];
}

// ---------------------------------------------------------------- launch counter
struct LaunchCounter {
    int64_t n = 0;
};

// ---------------------------------------------------------------- kernels (elementwise.cu)
int launch_resize_bilinear_tf1(const float* x, float* y, int B, int H, int W, int C, int oh, int ow, cudaStream_t s);
int launch_maxpool_f32(const float* x, float* y, int B, int H, int W, int C, cudaStream_t s);
// gradient of the 2x2 / 2 VALID max-pool: dy [B,H/2,W/2,C] -> dx [B,H,W,C], each window's gradient to its first maximum (row-major)
int launch_maxpool_backward_f32(const float* x, const float* dy, float* dx, int B, int H, int W, int C, cudaStream_t s);
int launch_maxpool_split(Split x, Split y, int B, int H, int W, int C, Half16 t, cudaStream_t s);
int launch_avgpool8(const float* x, float* y, int B, int H, int W, int C, cudaStream_t s);
int launch_f32_to_split(const float* x, Split y, int64_t rows, int C, int Cpad, Half16 t, cudaStream_t s);
int launch_split_to_f32(Split x, float* y, int64_t rows, int C, int Cpad, Half16 t, cudaStream_t s);
// seg post-process: scratch must hold seg_scratch_bytes(B,H,W) bytes (zeroed by the launcher).
int64_t seg_scratch_bytes(int B, int H, int W);
int launch_seg_postprocess(const float* logits, int B, int H, int W, void* scratch, uint8_t* hand_mask,
                           int32_t* max_loc, float* center, float* crop_size, float* scale_crop, cudaStream_t s,
                           int* n_launch, const float* low = nullptr, int LH = 0, int LW = 0);
int launch_crop_image(const float* image, const float* center, const float* scale, float* out, int B, int H, int W,
                      int C, int crop, cudaStream_t s);
int64_t argmax_scratch_bytes(int B, int C);
int launch_detect_keypoints(const float* sm, int B, int H, int W, int C, void* scratch, int32_t* uv, cudaStream_t s,
                            int* n_launch);
// fused x8 up-sampling of a [B,H,W,21] score map + per-channel arg-max (scratch: argmax_scratch_bytes(B, 21))
int launch_resize_argmax21(const float* x, float* y, int B, int H, int W, int oh, int ow, void* scratch, int32_t* uv, cudaStream_t s,
                           int* n_launch);
// dst[r, dst_off + c] = src[r, c] for c < C (fp32 channel copy into a wider NHWC tensor)
int launch_copy_channels(const float* src, float* dst, int64_t rows, int C, int dst_total, int dst_off, cudaStream_t s);
int launch_decode_records(const uint8_t* rec, int64_t record_bytes, int header_floats, int64_t image_off, int H, int W, int step,
                          int64_t mask_off, int tail_bytes, float* header, float* image, uint8_t* mask, uint8_t* tail, int B,
                          cudaStream_t s);
int launch_eval_dist(const float* gt, const uint8_t* vis, const float* pred, int n, int D, float* dist, cudaStream_t s);
int launch_gather_records_p2p(const float* coord3d, const int32_t* uv, const float* center, const float* scale, int B,
                              const uint64_t* peer_buffers, const uint64_t* peer_signals, uint64_t multicast_ptr, int rank, int world,
                              uint32_t epoch, int64_t parity_stride_floats, int max_batch, int* err_flag, cudaStream_t s);
int launch_pack_records(const float* coord3d, const int32_t* uv, const float* center, const float* scale, int B, float* out, cudaStream_t s);
int launch_mask_bbox(const float* mask, int B, int H, int W, float* center, float* bb, float* crop_size, cudaStream_t s);
int launch_leaky_relu(const float* x, float* y, int64_t n, cudaStream_t s);
int launch_flip_right_hand(const float* xyz, const uint8_t* cond_right, int B, float* out, cudaStream_t s);
int launch_bone_rel_trafo_inv(const float* rel, float* xyz, int B, cudaStream_t s);
int launch_rotate_canonical(const float* coord_can, const float* uxyz, const float* hand_side, int B, float* rot,
                            float* out, cudaStream_t s);

// ---------------------------------------------------------------- kernels (reader.cu): the dataset readers' forward generators
int launch_rhd_items(const float* header, const uint8_t* parts, const uint8_t* vis, int B, int use_wrist, int hand_crop, int crop_size,
                     float* xyz21, float* uv21, uint8_t* vis21, float* hand_side, float* kp_scale, float* xyz21_normed, float* crop_center,
                     float* crop_scale, float* cam_mat, cudaStream_t s);
int launch_stb_items(const float* header, int B, int use_wrist, float* xyz21, float* uv21, uint8_t* vis21, float* kp_scale, float* xyz21_normed,
                     cudaStream_t s);
int launch_gaussian_map(const float* coords_hw, const uint8_t* valid, int B, int N, int H, int W, float sigma, float* out, cudaStream_t s);
int launch_canonical_trafo(const float* xyz, const uint8_t* cond_right, int B, float* can, float* rot, float* rot_inv, cudaStream_t s);

// ---------------------------------------------------------------- kernels (conv_direct.cu)
struct DirectConvArgs {
    const float* x;       // [B,H,W,Cin_total] fp32, channels [cin_off, cin_off+Cin) are read
    int Cin_total, cin_off;
    const float* w;       // HWIO [k,k,Cin,Cout]
    const float* bias;    // [Cout]
    float* y;             // fp32 out (may be null) [B,Ho,Wo,Cout_total] at channel offset cout_off
    int Cout_total, cout_off;
    Split ys;             // optional split output [B,Ho,Wo,Cs_total] at channel offset cs_off
    int Cs_total, cs_off;
    Half16 half;
    int B, H, W, Cin, Cout, k, stride, leaky;
    float* splitk_scratch = nullptr;        // optional: enables deterministic split-K for layers with too few tiles
    int64_t splitk_scratch_floats = 0;
    int* err_flag = nullptr;                // forwarded to the tensor-core first-layer kernel (bounded barrier waits)
};
constexpr int64_t kConvSplitKScratchFloats = 600ll * 64 * 64;   // upper bound used by launch_conv_direct's split-K policy
int launch_conv_direct(const DirectConvArgs& a, cudaStream_t s);
int conv_direct_num_launches(const DirectConvArgs& a);   // 1, or 2 when the split-K policy applies
// scratch: fc_scratch_floats(B, in_f, out_f) floats (split-K partial sums); two kernels per call.  scratch_floats is the capacity
// of the scratch buffer: a call that would need more returns H3D_EINVAL and launches nothing.
int64_t fc_scratch_floats(int B, int in_f, int out_f);
int launch_fc(const float* x, const float* w, const float* bias, float* y, float* scratch, int64_t scratch_floats, int B, int in_f,
              int out_f, int leaky, int x_stride, cudaStream_t s);
// gathers [conv_feat(b, :feat) , hand_side(b, :2)] -> xcat [B, feat+2]
int launch_concat_handside(const float* feat, const float* hand_side, float* out, int B, int feat_n, cudaStream_t s);
// same as 16-bit split planes [B, Kpad] (Kpad % 64 == 0, zero padded): input of the tensor-core FC stack
int launch_concat_handside_split(const float* feat, const float* hand_side, Split out, int B, int feat_n, int Kpad, Half16 t, cudaStream_t s);

// ---------------------------------------------------------------- kernels (conv_wgmma.cu)
// first layer (Cin = 3, 3x3, 64 output channels) on the tensor cores, writing split planes (hi, lo optional)
int launch_conv_c3_tc(const float* x, const float* w, const float* bias, Split y, int Cs_total, int cs_off, int B, int H, int W, int leaky,
                      Half16 half, cudaStream_t s, int* err_flag = nullptr);
struct TcConvPlan;  // opaque: tensor maps + launch geometry of one tensor-core conv layer
struct TcConvDesc {
    // input activations (split planes) [B,H,W,Cin_total]; channels [0,Cin_pad) are read (Cin_pad % 64 == 0)
    Split x;
    int Cin_total, Cin_pad;
    // packed weights: [Cout_pad][k*k*Cin_pad] K-major 16-bit planes
    Split w;
    const float* bias;  // [Cout_pad] fp32
    const float* w_scale = nullptr;   // fp16 planes with passes 1 / 3: [Cout_pad] 2^-s un-doing the per-channel weight shift (split_fmt.cuh)
    int Cout, Cout_pad;
    // outputs: split planes at channel offset (16-byte aligned) and/or fp32
    Split y;
    int Cy_total, cy_off;
    float* yf;
    int Cyf_total, cyf_off;
    int B, H, W, k, leaky;
    int passes;  // 1, 3, or 4 = fp16 main pass + two fp8 (e4m3) correction passes (needs the l8 / h8 planes)
    float corr_scale = 0.f;   // passes == 4: 2^-(10 + b), un-does the scales of the fp8 operands (b: per-layer weight shift)
    Half16 half;
    int pool = 0;  // 1: fuse the following 2x2/2 max-pool; 2: stride-2 'SAME' convolution (even H, W); outputs are [B, H/2, W/2, C]
    int* err_flag = nullptr;   // device int: a barrier wait that times out stores its code here before trapping (h3d_ctx owns it)
    // conv1_1 fused into this layer: tc_conv_plan_create rejects it in the sm_90a build (tc_conv_can_fuse_first is false)
    const float* c1_w = nullptr; const float* c1_bias = nullptr; int c1_leaky = 0;
};
// Tuning switches: initialised from the environment once (H3D_TC_BN, H3D_FC_CHAIN, ...), changed only through tc_set_tuning().
struct TcTuning {
    // two_cta, c64, c64x2, pair128, stack, exp, c3_tma, c64_tma_out, chain, small_batch_split and fuse_c1 chose between kernel
    // variants of an earlier build; the sm_90a build has one convolution kernel family and accepts them without effect.
    int two_cta = -1;
    int bn = 0;            // 0 policy, else forced N tile (64 or 128)
    int c64 = 1, c64x2 = 1, pair128 = 1, stack = 1;
    int chunk_kb = 0;      // 0 policy, else K blocks per tensor-core partial sum
    int exp = 0;
    int no_side_stream = 0, no_pool_fusion = 0, lift_direct = 0;
    int c3_ffma = 0;       // 1: first layer on the register-tiled FFMA kernel instead of the tensor cores
    int no_seg_fusion = 0; // 1: HandSegNet's x8 up-sampling as its own launch (instead of fused into the mask post-processing)
    int c64_tma_out = 1;
    int fc_chain = 1;      // FC stacks + rotation epilogue of the lifting stage as one kernel (0 = one launch per layer)
    int fuse_c1 = 1;
    int small_batch_split = 1;
    int chain = 1;
    int pdl = 1;           // programmatic dependent launch between the tensor-core kernels (prologue overlaps the previous kernel's tail)
    int c3_tma = 1;
};
TcTuning& tc_tuning();
int tc_set_tuning(const char* key, int value);
// FC stack of a lifting network as ONE kernel (conv_wgmma.cu: fc_chain_kernel): up to 4 fully connected layers per chain, the
// activations of every layer as split planes [B, width_pad] (row stride = width rounded up to 64), the last layer fp32.
struct FcLayerDesc {
    Split x; int x_stride, in_features;      // input planes [B, x_stride], K = in_features rounded up to 64
    Split w; const float* bias; int out_features, out_pad;   // packed weights [out_pad][K] (pack_conv_weights with k = 1)
    const float* w_scale = nullptr;           // fp16 planes: per-output shifts (TcConvDesc::w_scale)
    Split y; int y_stride;                    // output planes (hidden layers) ...
    float* yf; int yf_stride;                 // ... or fp32 output (last layer)
    int leaky;
};
struct FcChainDesc { FcLayerDesc layer[4]; int num_layers = 0; };
struct FcChainPlan;
// chains: 1 (PosePrior only) or 2 (PosePrior, ViewpointNet + the fused Rodrigues / flip / rotate epilogue: can [B,63] and uxyz [B,3]
// are the fp32 outputs of the two chains, hand_side / rot / out are bound at launch time)
FcChainPlan* fc_chain_plan_create(const FcChainDesc* chains, int num_chains, int B, Half16 half, const float* can, const float* uxyz,
                                  unsigned int* counter, int* err_flag);
void fc_chain_plan_destroy(FcChainPlan* p);
int fc_chain_launch(const FcChainPlan* p, const float* hand_side, float* rot, float* out, cudaStream_t s);
TcConvPlan* tc_conv_plan_create(const TcConvDesc& d);   // nullptr on failure (h3d_last_error set)
void tc_conv_plan_destroy(TcConvPlan* p);
bool tc_conv_plan_chainable(const TcConvPlan* p);
int tc_conv_plan_signal_target(const TcConvPlan* p);
const TcConvDesc& tc_conv_plan_desc(const TcConvPlan* p);
void tc_conv_plan_set_chain(TcConvPlan* p, int* sched, const int* dep_cnt, int dep_target, int* sig_cnt);
int tc_conv_launch(const TcConvPlan* p, cudaStream_t s);
int tc_conv_launch_image(const TcConvPlan* p, const float* image, cudaStream_t s);   // plans with TcConvDesc::c1_w (none on sm_90a)
bool tc_conv_can_fuse_first(int H, int W, int Cin, int Cout, int k, int passes, int pool);
int64_t tc_conv_flops(const TcConvPlan* p);
int tc_num_sms();

// ---------------------------------------------------------------- kernels (conv_wgrad.cu): backward of the tensor-core convolution
// HWIO fp32 device weights -> 16-bit hi (/ lo) planes: forward [Cout_pad][k][k][Cin_pad] (as pack_conv_weights) or, with dgrad, the
// data-gradient operator [Cin_pad][k][k][Cout_pad] of the spatially flipped kernel; bias_pad [rows] = padded bias, or zeros with dgrad.
// w_scale [Cout_pad] (forward fp16 planes, else nullptr): the per-channel shift factors 2^-s of split_fmt.cuh, as the host packer
int launch_pack_conv_w(const float* w_hwio, const float* bias, Split out, float* bias_pad, float* w_scale, int k, int Cin, int Cout,
                       int Cin_pad, int Cout_pad, bool dgrad, Half16 half, cudaStream_t s);
// dy' = dy * act'(y) (y may be null without leaky) as bf16 split planes [B,H,W,Cout_pad] at the input resolution (stride 2: odd pixels);
// db_part (optional) [conv_grad_prep_blocks(B*H*W)][Cout_pad] per-block column sums for launch_bias_grad_reduce
int conv_grad_prep_blocks(int64_t pixels, int64_t* pixels_per_block);
int launch_conv_grad_prep(const float* dy, const float* y, Split out, float* db_part, int B, int H, int W, int Cout, int Cout_pad,
                          int stride, int leaky, cudaStream_t s);
int launch_bias_grad_reduce(const float* db_part, int nblk, int Cout, int Cout_pad, float* db, cudaStream_t s);
struct WgradDesc {
    Split x;        // input activations, split planes [B,H,W,Cin_pad]
    Split dy;       // dy' split planes [B,H,W,Cout_pad] (launch_conv_grad_prep)
    int B, H, W, Cin, Cout, Cin_pad, Cout_pad, k, passes;
    float* partial;  // conv_wgrad_partial_floats(...) floats of scratch
    float* dw;       // HWIO [k,k,Cin,Cout] fp32
    int* err_flag;
};
int64_t conv_wgrad_partial_floats(int B, int H, int W, int k, int Cin_pad, int Cout_pad);
int launch_conv_wgrad(const WgradDesc& d, cudaStream_t s);

// ---------------------------------------------------------------- kernels (train.cu): resize gradient, training losses, Adam
// scratch: resize_grad_scratch_floats(...) floats (the column pass's [B,oh,W,C] when both dimensions change); *n_launch kernels
int64_t resize_grad_scratch_floats(int B, int H, int W, int C, int oh, int ow);
int launch_resize_bilinear_tf1_grad(const float* dy, float* dx, float* scratch, int B, int H, int W, int C, int oh, int ow, cudaStream_t s,
                                    int* n_launch);
int64_t scoremap_loss_scratch_floats(int B, int H, int W);   // two kernels
int launch_scoremap_loss(const float* P, const float* T, const float* vis, float* scratch, int B, int H, int W, float* loss, float* rms,
                         cudaStream_t s);
int launch_scoremap_loss_grad(const float* P, const float* T, const float* vis, const float* rms, const float* grad, float* dP, int B,
                              int H, int W, cudaStream_t s);
int64_t softmax_xent_scratch_floats(int64_t rows);           // two kernels
int launch_softmax_xent(const float* logits, const float* labels, float* scratch, int64_t rows, float* loss, cudaStream_t s);
int launch_softmax_xent_grad(const float* logits, const float* labels, const float* grad, float* dlogits, int64_t rows, cudaStream_t s);
int launch_adam_step(const h3d_adam_tensor* table, int n, float* state, float beta1, float beta2, float epsilon, cudaStream_t s);
// mask bit 0: lr, bit 1: beta1_power, bit 2: beta2_power; the ticket is always cleared
int launch_adam_state_set(float* state, int mask, float lr, float beta1_power, float beta2_power, cudaStream_t s);

}  // namespace h3d

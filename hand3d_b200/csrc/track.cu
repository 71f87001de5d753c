// Frame-to-frame hand tracking (h3d_track_step): the crop of step t of a camera stream comes from the key-points step t - 1 found,
// following calc_center_bb (utils/general.py:271-328) and nets/ColorHandPose3DNetwork.py:82-85 with the 21 key-points in place of
// the hand mask.  Per slot b, in fp32, IEEE round-to-nearest and no contraction (DESIGN.md section 4.14):
//   p[k]    = (float(uv[k]) - 128) / scale + center        per axis (trafo_coords, utils/general.py:347-357, crop_size // 2 = 128)
//   center' = 0.5 (max_k p + min_k p),  size = max(extent_row, extent_col)
//   not finite -> the reference's fall-backs center (160, 160), size 100 (as mask_bbox_kernel)
//   scale'  = min(max(256 / (size * margin), 0.25), 5)
//   score   = (sum_k peak_k) / 21, peak_k = max of channel k of the last PoseNet2D stage's 32x32 map (NaN anywhere -> NaN)
//   lost    = (min_score is not NaN and !(score >= min_score)) or the fall-backs were used; a lost slot keeps its state's crop.
#include "common.cuh"

namespace h3d {

namespace {

constexpr int kTrackRows = 12;                    // threads per channel
constexpr int kTrackThreads = 21 * kTrackRows;    // 252: a multiple of 21, so thread t always reads channel t % 21 of the NHWC map
constexpr int kMapElems = 32 * 32 * 21;

// NaN-propagating max / min (numpy's np.max / np.min; fmaxf / fminf would drop a NaN)
__device__ __forceinline__ float nan_max(float m, float v) { return (v > m || v != v) ? v : m; }
__device__ __forceinline__ float nan_min(float m, float v) { return (v < m || v != v) ? v : m; }

__global__ void __launch_bounds__(kTrackThreads) track_update_kernel(const float* __restrict__ map, const int32_t* __restrict__ uv,
                                                                     const float* __restrict__ center, const float* __restrict__ scale,
                                                                     int B, float margin, float min_score, float* __restrict__ state) {
    __shared__ float s_part[kTrackRows][21];
    const int b = blockIdx.x, t = threadIdx.x;
    const float inf = __int_as_float(0x7f800000);
    // per-channel peaks: each thread reduces every 252nd element of the slot's map (all of channel t % 21), coalesced
    const float* m = map + (int64_t)b * kMapElems;
    float pk = -inf;
    for (int i = t; i < kMapElems; i += kTrackThreads) pk = nan_max(pk, __ldg(m + i));
    s_part[t / 21][t % 21] = pk;
    __syncthreads();
    if (t >= 32) return;
    // warp 0: lane k < 21 finishes peak k and handles key-point k
    const int k = t;
    float peak = -inf, pr = 0.f, pc = 0.f;
    if (k < 21) {
#pragma unroll
        for (int r = 0; r < kTrackRows; ++r) peak = nan_max(peak, s_part[r][k]);
        const float c0 = center[2 * b], c1 = center[2 * b + 1], sc = scale[b];
        pr = __fadd_rn(__fdiv_rn(__fsub_rn((float)uv[(int64_t)b * 42 + 2 * k], 128.0f), sc), c0);
        pc = __fadd_rn(__fdiv_rn(__fsub_rn((float)uv[(int64_t)b * 42 + 2 * k + 1], 128.0f), sc), c1);
    }
    float rmax = k < 21 ? pr : -inf, rmin = k < 21 ? pr : inf, cmax = k < 21 ? pc : -inf, cmin = k < 21 ? pc : inf;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        rmax = nan_max(rmax, __shfl_xor_sync(0xFFFFFFFFu, rmax, o)); rmin = nan_min(rmin, __shfl_xor_sync(0xFFFFFFFFu, rmin, o));
        cmax = nan_max(cmax, __shfl_xor_sync(0xFFFFFFFFu, cmax, o)); cmin = nan_min(cmin, __shfl_xor_sync(0xFFFFFFFFu, cmin, o));
    }
    // the sum over k in key-point order, from +0 (so that a -0 peak cannot leave a -0 score)
    float sum = 0.f;
    for (int j = 0; j < 21; ++j) sum = __fadd_rn(sum, __shfl_sync(0xFFFFFFFFu, peak, j));
    if (t != 0) return;
    const float score = __fdiv_rn(sum, 21.0f);
    float c0 = __fmul_rn(0.5f, __fadd_rn(rmax, rmin)), c1 = __fmul_rn(0.5f, __fadd_rn(cmax, cmin));
    float sz = fmaxf(__fsub_rn(rmax, rmin), __fsub_rn(cmax, cmin));
    const bool fallback = !(isfinite(c0) && isfinite(c1) && isfinite(sz));
    if (fallback) { c0 = 160.0f; c1 = 160.0f; sz = 100.0f; }
    const float sc = fminf(fmaxf(__fdiv_rn(256.0f, __fmul_rn(sz, margin)), 0.25f), 5.0f);
    const bool lost = fallback || (min_score == min_score && !(score >= min_score));
    float* st_center = state + (int64_t)H3D_TRACK_CENTER * B;
    if (!lost) {
        st_center[2 * b] = c0; st_center[2 * b + 1] = c1;
        state[(int64_t)H3D_TRACK_SCALE * B + b] = sc;
    }
    state[(int64_t)H3D_TRACK_SCORE * B + b] = score;
    reinterpret_cast<int32_t*>(state)[(int64_t)H3D_TRACK_LOST * B + b] = lost ? 1 : 0;
}

// Slot selection of a slots step (h3d_track_step_slots): one CTA walks the B slots in chunks of kSelThreads; a chunk's positions are an
// exclusive prefix sum of its flags (warp ballots, then the warp totals), added to the running count of the chunks before it.  So the
// selected slots land in ascending order and no atomic decides a position.  Reads the lost flags the previous step's update wrote.
constexpr int kSelThreads = 256;

__global__ void __launch_bounds__(kSelThreads) track_select_kernel(const int32_t* __restrict__ lost, const int32_t* __restrict__ force,
                                                                   int B, int32_t* __restrict__ sel, int32_t* __restrict__ detected) {
    __shared__ int s_warp[kSelThreads / 32];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    int32_t* slots = sel + 1;
    int32_t* pos = sel + 1 + B;
    int base = 0;
    for (int c0 = 0; c0 < B; c0 += kSelThreads) {
        const int b = c0 + t;
        const bool on = b < B && (lost[b] != 0 || (force && force[b] != 0));
        const unsigned m = __ballot_sync(0xFFFFFFFFu, on);
        if (lane == 0) s_warp[warp] = __popc(m);
        __syncthreads();
        int before = base, total = base;
        for (int w = 0; w < kSelThreads / 32; ++w) {
            if (w < warp) before += s_warp[w];
            total += s_warp[w];
        }
        const int p = before + __popc(m & ((1u << lane) - 1u));
        if (b < B) {
            pos[b] = on ? p : -1;
            if (on) slots[p] = b;
            if (detected) detected[b] = on ? 1 : 0;
        }
        base = total;
        __syncthreads();   // s_warp is rewritten by the next chunk
    }
    if (t == 0) sel[0] = base;
}

// The crop of a slots step: a selected slot takes the one its mask produced (compact index pos[b]), every other slot its state's crop.
__global__ void track_merge_kernel(const float* __restrict__ state, const int32_t* __restrict__ sel, const float* __restrict__ cen_c,
                                   const float* __restrict__ scl_c, int B, float* __restrict__ center, float* __restrict__ scale) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const int p = sel[1 + B + b];
    const float* st_center = state + (int64_t)H3D_TRACK_CENTER * B;
    if (p >= 0) {
        center[2 * b] = cen_c[2 * p]; center[2 * b + 1] = cen_c[2 * p + 1];
        scale[b] = scl_c[p];
    } else {
        center[2 * b] = st_center[2 * b]; center[2 * b + 1] = st_center[2 * b + 1];
        scale[b] = state[(int64_t)H3D_TRACK_SCALE * B + b];
    }
}

}  // namespace

int launch_track_select(const void* state, const int32_t* force, int B, int32_t* sel, int32_t* detected, cudaStream_t s) {
    const int32_t* lost = reinterpret_cast<const int32_t*>(state) + (int64_t)H3D_TRACK_LOST * B;
    track_select_kernel<<<1, kSelThreads, 0, s>>>(lost, force, B, sel, detected);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

int launch_track_merge(const void* state, const int32_t* sel, const float* cen_c, const float* scl_c, int B, float* center, float* scale,
                       cudaStream_t s) {
    track_merge_kernel<<<ceil_div(B, 128), 128, 0, s>>>((const float*)state, sel, cen_c, scl_c, B, center, scale);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

int launch_track_update(const float* map32, const int32_t* uv, const float* center, const float* scale, int B, float margin,
                        float min_score, void* state, cudaStream_t s) {
    track_update_kernel<<<B, kTrackThreads, 0, s>>>(map32, uv, center, scale, B, margin, min_score, (float*)state);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

}  // namespace h3d

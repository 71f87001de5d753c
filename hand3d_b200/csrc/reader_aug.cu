// Training-mode augmentation of the RHD reader (data/BinaryDbReader.py:160-401): the per-sample random parameters and the one pass
// over the image that applies tf.image.random_hue and / or the random_crop window.  The generator, the counter layout and the
// parameter layout are documented with the H3D_AUG_* defines in include/hand3d_b200.h.  The coordinate / crop noises are applied by
// rhd_items_kernel and the score-map dropout by gaussian_map_kernel<true> (reader.cu), both from the same parameter tensor.
#include "common.cuh"
#include "philox.cuh"

namespace h3d {

__device__ __forceinline__ void draw(uint64_t seed, uint64_t serial, uint64_t vid, uint64_t attempt, uint64_t w[4]) {
    w[0] = serial; w[1] = vid; w[2] = attempt; w[3] = 0;
    philox4x64_10(w, seed, H3D_AUG_STREAM_ITEMS);
}

// TF's random_uniform affine step in fp32: u * (max - min) + min, without contraction.
__device__ __forceinline__ float uniform_range(float u, float lo, float hi) { return __fadd_rn(__fmul_rn(u, __fsub_rn(hi, lo)), lo); }

// Standard normal truncated to [-2, 2] (tf.truncated_normal's support): Box-Muller in fp64, first accepted value of z0, z1 per attempt.
__device__ float truncated_normal(uint64_t seed, uint64_t serial, uint64_t vid) {
    for (int a = 0; a < H3D_AUG_MAX_ATTEMPTS; ++a) {
        uint64_t w[4];
        draw(seed, serial, vid, (uint64_t)a, w);
        const double u1 = (double)((w[0] >> 11) + 1) * 0x1p-53, u2 = (double)(w[1] >> 11) * 0x1p-53;
        const double r = sqrt(__dmul_rn(-2.0, log(u1)));
        double sn, cs;
        sincospi(__dmul_rn(2.0, u2), &sn, &cs);
        const float z0 = (float)__dmul_rn(r, cs), z1 = (float)__dmul_rn(r, sn);
        if (fabsf(z0) <= 2.f) return z0;
        if (fabsf(z1) <= 2.f) return z1;
    }
    return 0.f;                                      // all 2 * H3D_AUG_MAX_ATTEMPTS draws rejected: p ~ 0.0455^32
}

// One thread per (sample, parameter slot): the final value (px, factor, offset, bit) of each flag that is on, neutral values otherwise.
__global__ void aug_params_kernel(const int64_t* __restrict__ serials, int B, uint64_t seed, int flags, float* __restrict__ params) {
    const int b = blockIdx.x, j = threadIdx.x;
    if (b >= B || j >= H3D_AUG_PARAMS) return;
    const uint64_t serial = (uint64_t)serials[b];
    float v = 0.f;
    auto tn = [&](float sigma) { return __fadd_rn(__fmul_rn(truncated_normal(seed, serial, (uint64_t)j), sigma), 0.f); };   // z * stddev + mean
    uint64_t w[4];
    if (j < H3D_AUG_CENTER_NOISE) {
        if (flags & H3D_AUG_COORD_UV_NOISE) v = tn(2.5f);
    } else if (j < H3D_AUG_SCALE) {
        if (flags & H3D_AUG_CROP_CENTER_NOISE) v = tn(20.0f);
    } else if (j == H3D_AUG_SCALE) {
        v = 1.f;
        if (flags & H3D_AUG_CROP_SCALE_NOISE) { draw(seed, serial, j, 0, w); v = uniform_range(uniform01(w[0]), 1.0f, 1.2f); }
    } else if (j < H3D_AUG_HUE_DELTA) {
        if (flags & H3D_AUG_CROP_OFFSET_NOISE) v = tn(10.0f);
    } else if (j == H3D_AUG_HUE_DELTA) {
        if (flags & H3D_AUG_HUE) { draw(seed, serial, j, 0, w); v = uniform_range(uniform01(w[0]), -0.1f, 0.1f); }
    } else if (j < H3D_AUG_KEEP) {
        if (flags & H3D_AUG_RANDOM_CROP) { draw(seed, serial, j, 0, w); v = (float)(w[0] % 65ull); }    // random_crop: [0, 320 - 256]
    } else if (j < H3D_AUG_USED) {
        v = 1.f;
        if (flags & H3D_AUG_SCOREMAP_DROPOUT) { draw(seed, serial, j, 0, w); v = floorf(__fadd_rn(0.8f, uniform01(w[0]))); }
    }
    params[(int64_t)b * H3D_AUG_PARAMS + j] = v;
}

int launch_reader_aug_params(const int64_t* serials, int B, uint64_t seed, int flags, float* params, cudaStream_t s) {
    aug_params_kernel<<<B, H3D_AUG_PARAMS, 0, s>>>(serials, B, seed, flags, params);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

// ------------------------------------------------------------------------------------------ shuffle queue
// The windowed shuffle of shuffle_batch_join(capacity=100, min_after_dequeue=50) on the device (state layout with H3D_READER_STATE_*).
// Dequeue n reads word n of Philox4x64-10 keyed (seed, H3D_AUG_STREAM_SHUFFLE) in numpy.random.Philox.random_raw order: numpy bumps
// its 256-bit counter BEFORE it fills its 4-word buffer, so word n is word (n mod 4) of the block at counter (n / 4 + 1, 0, 0, 0).
// The slot choices are independent of each other and are drawn in parallel; taking and refilling the slots is sequential (thread 0).
constexpr int kQueueChunk = 128;
__global__ void __launch_bounds__(kQueueChunk) next_serials_kernel(int64_t* __restrict__ state, int B, uint64_t seed, int shuffle,
                                                                   int64_t* __restrict__ serials) {
    __shared__ int64_t s_slot[H3D_READER_QUEUE_CAPACITY];
    __shared__ int s_k[kQueueChunk];
    const uint64_t n0 = (uint64_t)state[H3D_READER_STATE_COUNT];
    int64_t next = state[H3D_READER_STATE_NEXT];
    if (!shuffle) {                                  // the in-order stream: consecutive positions
        for (int i = threadIdx.x; i < B; i += blockDim.x) serials[i] = next + i;
        __syncthreads();                             // every thread has read the state before it moves
        if (threadIdx.x == 0) { state[H3D_READER_STATE_COUNT] = (int64_t)(n0 + (uint64_t)B); state[H3D_READER_STATE_NEXT] = next + B; }
        return;
    }
    for (int i = threadIdx.x; i < H3D_READER_QUEUE_CAPACITY; i += blockDim.x) s_slot[i] = state[H3D_READER_STATE_SLOTS + i];
    for (int base = 0; base < B; base += kQueueChunk) {
        const int i = base + threadIdx.x;
        if (i < B) {
            const uint64_t n = n0 + (uint64_t)i;
            uint64_t c[4] = {(n >> 2) + 1, 0, 0, 0};
            philox4x64_10(c, seed, H3D_AUG_STREAM_SHUFFLE);
            const int j = (int)(n & 3);
            const uint64_t w = j == 0 ? c[0] : j == 1 ? c[1] : j == 2 ? c[2] : c[3];
            s_k[threadIdx.x] = (int)(w % (uint64_t)H3D_READER_QUEUE_CAPACITY);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            const int m = min(kQueueChunk, B - base);
            for (int t = 0; t < m; ++t) {
                const int k = s_k[t];
                serials[base + t] = s_slot[k];
                s_slot[k] = next++;
            }
        }
        __syncthreads();
    }
    for (int i = threadIdx.x; i < H3D_READER_QUEUE_CAPACITY; i += blockDim.x) state[H3D_READER_STATE_SLOTS + i] = s_slot[i];
    if (threadIdx.x == 0) { state[H3D_READER_STATE_COUNT] = (int64_t)(n0 + (uint64_t)B); state[H3D_READER_STATE_NEXT] = next; }
}

int launch_reader_next_serials(int64_t* state, int B, uint64_t seed, int shuffle, int64_t* serials, cudaStream_t s) {
    next_serials_kernel<<<1, kQueueChunk, 0, s>>>(state, B, seed, shuffle, serials);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

// ------------------------------------------------------------------------------------------ adjust_hue (TF 1.3, non-fused)
// rgb_to_hsv / hsv_to_rgb as TF's colorspace_op.h functors evaluate them, element by element in fp32, then h = mod(h + (delta + 1), 1)
// between them (image_ops_impl.adjust_hue).  S = V > 0 ? range / V : 0, so a pixel whose largest channel is <= 0 -- every dark pixel
// of the reader's image / 255 - 0.5 -- comes back grey (R = G = B = V).
__device__ __forceinline__ void adjust_hue_tf13(float& r, float& g, float& b, float delta_p1) {
    const float v = fmaxf(fmaxf(r, g), b);
    const float range = __fsub_rn(v, fminf(fminf(r, g), b));
    const float s = v > 0.f ? __fdiv_rn(range, v) : 0.f;
    float h = 0.f;
    if (range > 0.f) {
        const float norm = __fmul_rn(__frcp_rn(range), 1.f / 6.f);
        if (r == v) h = __fmul_rn(norm, __fsub_rn(g, b));
        else if (g == v) h = __fadd_rn(__fmul_rn(norm, __fsub_rn(b, r)), 2.f / 6.f);
        else h = __fadd_rn(__fmul_rn(norm, __fsub_rn(r, g)), 4.f / 6.f);
    }
    if (h < 0.f) h = __fadd_rn(h, 1.f);
    h = fmodf(__fadd_rn(h, delta_p1), 1.f);          // exact; the argument is positive
    const float dh = __fmul_rn(h, 6.f);
    const float dr = fminf(fmaxf(__fsub_rn(fabsf(__fsub_rn(dh, 3.f)), 1.f), 0.f), 1.f);
    const float dg = fminf(fmaxf(__fadd_rn(-fabsf(__fsub_rn(dh, 2.f)), 2.f), 0.f), 1.f);
    const float db = fminf(fmaxf(__fadd_rn(-fabsf(__fsub_rn(dh, 4.f)), 2.f), 0.f), 1.f);
    const float one_s = __fadd_rn(-s, 1.f);
    r = __fmul_rn(__fadd_rn(one_s, __fmul_rn(s, dr)), v);
    g = __fmul_rn(__fadd_rn(one_s, __fmul_rn(s, dg)), v);
    b = __fmul_rn(__fadd_rn(one_s, __fmul_rn(s, db)), v);
}

// One thread per output pixel of sample blockIdx.y: the (optionally hue-shifted) pixel at (y + oy, x + ox), and with the window the
// hand_parts / hand_mask values at the same place (tf.random_crop of the stacked [image, parts, mask] tensor, :383-392).
__global__ void augment_image_kernel(const float* __restrict__ image, const uint8_t* __restrict__ parts, const float* __restrict__ params,
                                     int H, int W, int flags, int oh, int ow, float* __restrict__ out_image, int32_t* __restrict__ out_parts,
                                     int32_t* __restrict__ out_mask) {
    const int b = blockIdx.y;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)oh * ow) return;
    const int y = (int)(i / ow), x = (int)(i - (int64_t)y * ow);
    const float* prm = params + (int64_t)b * H3D_AUG_PARAMS;
    int oy = 0, ox = 0;
    if (flags & H3D_AUG_RANDOM_CROP) {               // clamped so that caller-supplied parameters cannot read outside the image
        oy = min(max((int)prm[H3D_AUG_WINDOW], 0), H - oh); ox = min(max((int)prm[H3D_AUG_WINDOW + 1], 0), W - ow);
    }
    const int64_t src = (int64_t)b * H * W + (int64_t)(y + oy) * W + (x + ox);
    float r = image[3 * src], g = image[3 * src + 1], bl = image[3 * src + 2];
    if (flags & H3D_AUG_HUE) adjust_hue_tf13(r, g, bl, __fadd_rn(prm[H3D_AUG_HUE_DELTA], 1.f));
    const int64_t dst = (int64_t)b * oh * ow + i;
    out_image[3 * dst] = r; out_image[3 * dst + 1] = g; out_image[3 * dst + 2] = bl;
    if (parts && (out_parts || out_mask)) {
        const int p = parts[src];
        if (out_parts) out_parts[dst] = p;
        if (out_mask) { out_mask[2 * dst] = p > 1 ? 0 : 1; out_mask[2 * dst + 1] = p > 1 ? 1 : 0; }
    }
}

int launch_augment_image(const float* image, const uint8_t* parts, const float* params, int B, int H, int W, int flags, int window,
                         float* out_image, int32_t* out_parts, int32_t* out_mask, cudaStream_t s) {
    const bool crop = flags & H3D_AUG_RANDOM_CROP;
    H3D_REQUIRE(!crop || (window > 0 && H - window == 64 && W - window == 64), "augment_image: the window must be 64 px smaller than the image "
                "in both axes (random_crop offsets lie in [0, 64])");
    const int oh = crop ? window : H, ow = crop ? window : W;
    dim3 grid((unsigned)ceil_div64((int64_t)oh * ow, 256), B);
    augment_image_kernel<<<grid, 256, 0, s>>>(image, parts, params, H, W, flags, oh, ow, out_image, out_parts, out_mask);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

}  // namespace h3d

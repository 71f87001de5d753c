// HBM-bound kernels of the ColorHandPose3D forward pass: TF1-legacy bilinear resize, 2x2 max-pool,
// 8x8 avg-pool, soft-max / round / arg-max + 32-pass geodesic mask growing + bounding box,
// crop_and_resize, per-channel heat-map arg-max, Rodrigues / flip / rotate epilogue.
//
// All arithmetic that feeds a discrete decision or an interpolated output uses explicit
// __fmul_rn/__fadd_rn/__fsub_rn so that nvcc cannot contract to FMA: the TF-1.3 CPU kernels the
// oracle restates use separate multiply and add (SURVEY.md section 9).
#include "common.cuh"
#include "split_fmt.cuh"

namespace h3d {

__device__ __forceinline__ float lerp_tf(float a, float b, float t) {
    // a + (b - a) * t  without FMA contraction (TF compute_lerp)
    return __fadd_rn(a, __fmul_rn(__fsub_rn(b, a), t));
}

// =============================================================================================
// tf.image.resize_images bilinear, align_corners=False, legacy (nets/ColorHandPose3DNetwork.py:97,128,166)
// One thread produces 4 consecutive floats of the flattened (ox, c) output row -> float4 stores.
// =============================================================================================
// CT > 0: channel count known at compile time (2 and 21 on the hot path) -> the per-element e / C becomes a multiply-shift.
template <int CT>
__global__ void resize_bilinear_tf1_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H, int W,
                                           int C_rt, int oh, int ow, float hscale, float wscale) {
    const int C = CT > 0 ? CT : C_rt;
    const int row_elems = ow * C;
    const int vec_per_row = (row_elems + 3) >> 2;
    const int64_t total = (int64_t)B * oh * vec_per_row;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int v = (int)(i % vec_per_row);
        const int oy = (int)((i / vec_per_row) % oh);
        const int b = (int)(i / ((int64_t)vec_per_row * oh));
        const float in_y = __fmul_rn((float)oy, hscale);
        const int y0 = (int)floorf(in_y);
        const int y1 = min(y0 + 1, H - 1);
        const float ly = __fsub_rn(in_y, (float)y0);
        const float* r0 = x + ((int64_t)b * H + y0) * W * C;
        const float* r1 = x + ((int64_t)b * H + y1) * W * C;
        float out[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int e = v * 4 + j;
            if (e < row_elems) {
                const int ox = e / C, c = e - ox * C;
                const float in_x = __fmul_rn((float)ox, wscale);
                const int x0 = (int)floorf(in_x);
                const int x1 = min(x0 + 1, W - 1);
                const float lx = __fsub_rn(in_x, (float)x0);
                const float tl = __ldg(r0 + x0 * C + c), tr = __ldg(r0 + x1 * C + c);
                const float bl = __ldg(r1 + x0 * C + c), br = __ldg(r1 + x1 * C + c);
                const float top = lerp_tf(tl, tr, lx);
                const float bot = lerp_tf(bl, br, lx);
                out[j] = lerp_tf(top, bot, ly);
            } else {
                out[j] = 0.f;
            }
        }
        float* dst = y + ((int64_t)b * oh + oy) * row_elems + v * 4;
        if ((row_elems & 3) == 0) {
            *reinterpret_cast<float4*>(dst) = make_float4(out[0], out[1], out[2], out[3]);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (v * 4 + j < row_elems) dst[j] = out[j];
        }
    }
}

int launch_resize_bilinear_tf1(const float* x, float* y, int B, int H, int W, int C, int oh, int ow, cudaStream_t s) {
    if (H == oh && W == ow) {  // TF returns the input unchanged when the size already matches
        H3D_CUDA(cudaMemcpyAsync(y, x, (size_t)B * H * W * C * sizeof(float), cudaMemcpyDeviceToDevice, s));
        return H3D_OK;
    }
    const float hscale = (float)H / (float)oh, wscale = (float)W / (float)ow;
    const int64_t total = (int64_t)B * oh * ((ow * C + 3) / 4);
    const int threads = 256;
    const int blocks = (int)std::min<int64_t>(ceil_div64(total, threads), 132 * 32);
    if (C == 21) resize_bilinear_tf1_kernel<21><<<blocks, threads, 0, s>>>(x, y, B, H, W, C, oh, ow, hscale, wscale);
    else if (C == 2) resize_bilinear_tf1_kernel<2><<<blocks, threads, 0, s>>>(x, y, B, H, W, C, oh, ow, hscale, wscale);
    else resize_bilinear_tf1_kernel<0><<<blocks, threads, 0, s>>>(x, y, B, H, W, C, oh, ow, hscale, wscale);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

// =============================================================================================
// NetworkOps.max_pool 2x2/2 VALID (utils/general.py:62-65)
// =============================================================================================
__global__ void maxpool_f32_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H, int W, int C) {
    const int Ho = H >> 1, Wo = W >> 1;
    const int C4 = C >> 2;
    const int64_t total = (int64_t)B * Ho * Wo * C4;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c4 = (int)(i % C4);
        const int ox = (int)((i / C4) % Wo);
        const int oy = (int)((i / ((int64_t)C4 * Wo)) % Ho);
        const int b = (int)(i / ((int64_t)C4 * Wo * Ho));
        const float4* p = reinterpret_cast<const float4*>(x + (((int64_t)b * H + 2 * oy) * W + 2 * ox) * C) + c4;
        const float4 a = __ldg(p), bq = __ldg(p + C4), c = __ldg(p + (int64_t)W * C4), d = __ldg(p + (int64_t)W * C4 + C4);
        float4 r;
        r.x = fmaxf(fmaxf(a.x, bq.x), fmaxf(c.x, d.x));
        r.y = fmaxf(fmaxf(a.y, bq.y), fmaxf(c.y, d.y));
        r.z = fmaxf(fmaxf(a.z, bq.z), fmaxf(c.z, d.z));
        r.w = fmaxf(fmaxf(a.w, bq.w), fmaxf(c.w, d.w));
        reinterpret_cast<float4*>(y)[i] = r;
    }
}

__global__ void maxpool_f32_scalar_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H, int W, int C) {
    const int Ho = H >> 1, Wo = W >> 1;
    const int64_t total = (int64_t)B * Ho * Wo * C;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const int ox = (int)((i / C) % Wo);
        const int oy = (int)((i / ((int64_t)C * Wo)) % Ho);
        const int b = (int)(i / ((int64_t)C * Wo * Ho));
        const float* p = x + (((int64_t)b * H + 2 * oy) * W + 2 * ox) * C + c;
        y[i] = fmaxf(fmaxf(p[0], p[C]), fmaxf(p[(int64_t)W * C], p[(int64_t)W * C + C]));
    }
}

int launch_maxpool_f32(const float* x, float* y, int B, int H, int W, int C, cudaStream_t s) {
    const int threads = 256;
    if ((C & 3) == 0) {
        const int64_t total = (int64_t)B * (H / 2) * (W / 2) * (C / 4);
        maxpool_f32_kernel<<<(int)std::min<int64_t>(ceil_div64(total, threads), 132 * 32), threads, 0, s>>>(x, y, B, H, W, C);
    } else {
        const int64_t total = (int64_t)B * (H / 2) * (W / 2) * C;
        maxpool_f32_scalar_kernel<<<(int)std::min<int64_t>(ceil_div64(total, threads), 132 * 32), threads, 0, s>>>(x, y, B, H, W, C);
    }
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

// Gradient of NetworkOps.max_pool: one thread per (window, channel) writes the window's four dx values; the gradient goes to the first
// maximum in row-major window order (TF's CPU MaxPoolGrad).  Odd trailing rows / columns (dropped by VALID) are zeroed by the launcher.
__global__ void maxpool_backward_f32_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dx, int B, int H,
                                            int W, int C) {
    const int Ho = H >> 1, Wo = W >> 1;
    const int64_t total = (int64_t)B * Ho * Wo * C;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const int ox = (int)((i / C) % Wo);
        const int oy = (int)((i / ((int64_t)C * Wo)) % Ho);
        const int b = (int)(i / ((int64_t)C * Wo * Ho));
        const int64_t base = (((int64_t)b * H + 2 * oy) * W + 2 * ox) * C + c;
        const int64_t offs[4] = {0, C, (int64_t)W * C, (int64_t)W * C + C};
        int arg = 0;
        float best = __ldg(x + base);
#pragma unroll
        for (int q = 1; q < 4; ++q) {
            const float v = __ldg(x + base + offs[q]);
            if (v > best) { best = v; arg = q; }
        }
        const float g = __ldg(dy + i);
#pragma unroll
        for (int q = 0; q < 4; ++q) dx[base + offs[q]] = q == arg ? g : 0.f;
    }
}

int launch_maxpool_backward_f32(const float* x, const float* dy, float* dx, int B, int H, int W, int C, cudaStream_t s) {
    if ((H | W) & 1) H3D_CUDA(cudaMemsetAsync(dx, 0, (size_t)B * H * W * C * sizeof(float), s));
    const int64_t total = (int64_t)B * (H / 2) * (W / 2) * C;
    if (total == 0) return H3D_OK;
    maxpool_backward_f32_kernel<<<(int)std::min<int64_t>(ceil_div64(total, 256), 132 * 32), 256, 0, s>>>(x, dy, dx, B, H, W, C);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

template <bool FP16>
__device__ __forceinline__ float h16_to_f32(uint16_t v) {
    if (FP16) return __half2float(__ushort_as_half(v));
    return __uint_as_float((uint32_t)v << 16);
}
template <bool FP16>
__device__ __forceinline__ uint16_t f32_to_h16(float v) {
    if (FP16) return __half_as_ushort(__float2half_rn(v));
    return __bfloat16_as_ushort(__float2bfloat16_rn(v));
}

// Split-format 2x2 max-pool: 8 channels (one uint4 per plane) per thread.  The arg-max element's
// (hi, lo) pair is carried through unchanged, so the pooled value is exactly one of the inputs.
template <bool FP16, bool HAS_LO>
__global__ void maxpool_split_kernel(const uint4* __restrict__ xh, const uint4* __restrict__ xl, uint4* __restrict__ yh,
                                     uint4* __restrict__ yl, int B, int H, int W, int C8) {
    const int Ho = H >> 1, Wo = W >> 1;
    const int64_t total = (int64_t)B * Ho * Wo * C8;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c8 = (int)(i % C8);
        const int ox = (int)((i / C8) % Wo);
        const int oy = (int)((i / ((int64_t)C8 * Wo)) % Ho);
        const int b = (int)(i / ((int64_t)C8 * Wo * Ho));
        const int64_t base = (((int64_t)b * H + 2 * oy) * W + 2 * ox) * C8 + c8;
        const int64_t offs[4] = {0, C8, (int64_t)W * C8, (int64_t)W * C8 + C8};
        uint16_t bh[8], bl[8];
        float bv[8];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const uint4 vh = __ldg(xh + base + offs[q]);
            uint4 vl = make_uint4(0, 0, 0, 0);
            if (HAS_LO) vl = __ldg(xl + base + offs[q]);
            const uint16_t* ph = reinterpret_cast<const uint16_t*>(&vh);
            const uint16_t* pl = reinterpret_cast<const uint16_t*>(&vl);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float v = h16_to_f32<FP16>(ph[j]);
                if (HAS_LO) v += h16_to_f32<FP16>(pl[j]);
                if (q == 0 || v > bv[j]) { bv[j] = v; bh[j] = ph[j]; bl[j] = pl[j]; }
            }
        }
        yh[i] = *reinterpret_cast<uint4*>(bh);
        if (HAS_LO) yl[i] = *reinterpret_cast<uint4*>(bl);
    }
}

int launch_maxpool_split(Split x, Split y, int B, int H, int W, int C, Half16 t, cudaStream_t s) {
    H3D_REQUIRE((C & 7) == 0, "maxpool_split: C %% 8 != 0");
    const int threads = 256;
    const int64_t total = (int64_t)B * (H / 2) * (W / 2) * (C / 8);
    const int blocks = (int)std::min<int64_t>(ceil_div64(total, threads), 132 * 32);
    const uint4 *xh = (const uint4*)x.hi, *xl = (const uint4*)x.lo;
    uint4 *yh = (uint4*)y.hi, *yl = (uint4*)y.lo;
    const bool lo = x.lo != nullptr;
    if (t == Half16::FP16) {
        if (lo) maxpool_split_kernel<true, true><<<blocks, threads, 0, s>>>(xh, xl, yh, yl, B, H, W, C / 8);
        else maxpool_split_kernel<true, false><<<blocks, threads, 0, s>>>(xh, xl, yh, yl, B, H, W, C / 8);
    } else {
        if (lo) maxpool_split_kernel<false, true><<<blocks, threads, 0, s>>>(xh, xl, yh, yl, B, H, W, C / 8);
        else maxpool_split_kernel<false, false><<<blocks, threads, 0, s>>>(xh, xl, yh, yl, B, H, W, C / 8);
    }
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

// =============================================================================================
// tf.nn.avg_pool 8x8/8 (nets/PosePriorNetwork.py:61)
// =============================================================================================
__global__ void avgpool8_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H, int W, int C) {
    const int Ho = H / 8, Wo = W / 8;
    const int64_t total = (int64_t)B * Ho * Wo * C;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const int ox = (int)((i / C) % Wo);
        const int oy = (int)((i / ((int64_t)C * Wo)) % Ho);
        const int b = (int)(i / ((int64_t)C * Wo * Ho));
        const float* p = x + (((int64_t)b * H + 8 * oy) * W + 8 * ox) * C + c;
        float acc = 0.f;
        for (int dy = 0; dy < 8; ++dy)
            for (int dx = 0; dx < 8; ++dx) acc += __ldg(p + ((int64_t)dy * W + dx) * C);
        y[i] = acc / 64.0f;
    }
}

int launch_avgpool8(const float* x, float* y, int B, int H, int W, int C, cudaStream_t s) {
    H3D_REQUIRE(H % 8 == 0 && W % 8 == 0, "avgpool8: H, W must be multiples of 8");
    const int64_t total = (int64_t)B * (H / 8) * (W / 8) * C;
    avgpool8_kernel<<<(int)std::min<int64_t>(ceil_div64(total, 256), 132 * 32), 256, 0, s>>>(x, y, B, H, W, C);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

// =============================================================================================
// fp32 <-> split conversions (operator-level tensor-core entry point / tests)
// =============================================================================================
template <bool FP16>
__global__ void f32_to_split_kernel(const float* __restrict__ x, uint16_t* __restrict__ hi, uint16_t* __restrict__ lo,
                                    int64_t rows, int C, int Cpad) {
    const int64_t total = rows * Cpad;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % Cpad);
        const int64_t r = i / Cpad;
        const float v = c < C ? x[r * C + c] : 0.f;
        const uint16_t h = f32_to_h16<FP16>(v);
        hi[i] = h;
        if (lo) lo[i] = f32_to_h16<FP16>(v - h16_to_f32<FP16>(h));
    }
}
template <bool FP16>
__global__ void split_to_f32_kernel(const uint16_t* __restrict__ hi, const uint16_t* __restrict__ lo, float* __restrict__ y,
                                    int64_t rows, int C, int Cpad) {
    const int64_t total = rows * C;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const int64_t r = i / C;
        float v = h16_to_f32<FP16>(hi[r * Cpad + c]);
        if (lo) v += h16_to_f32<FP16>(lo[r * Cpad + c]);
        y[i] = v;
    }
}
__global__ void f32_to_f8c_kernel(const float* __restrict__ x, uint16_t* __restrict__ h16, uint8_t* __restrict__ l8, uint8_t* __restrict__ h8,
                                  int64_t rows, int C, int Cpad) {
    const int64_t total = rows * Cpad;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % Cpad);
        const F8cPlanes p = f32_to_f8c(c < C ? x[(i / Cpad) * C + c] : 0.f);
        h16[i] = p.h16; l8[i] = p.l8; h8[i] = p.h8;
    }
}
__global__ void f8c_to_f32_kernel(const uint16_t* __restrict__ h16, const uint8_t* __restrict__ l8, float* __restrict__ y, int64_t rows, int C,
                                  int Cpad) {
    const int64_t total = rows * C;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t j = (i / C) * Cpad + (i % C);
        y[i] = __half2float(__ushort_as_half(h16[j])) * (1.0f / kF8XMainScale) + e4m3_to_f32(l8[j]) * (1.0f / kF8XLoScale);
    }
}

int launch_f32_to_split(const float* x, Split y, int64_t rows, int C, int Cpad, Half16 t, cudaStream_t s) {
    if (y.l8) {
        f32_to_f8c_kernel<<<(int)std::min<int64_t>(ceil_div64(rows * Cpad, 256), 132 * 32), 256, 0, s>>>(x, y.hi, y.l8, y.h8, rows, C, Cpad);
        H3D_CHECK_LAUNCH();
        return H3D_OK;
    }
    const int blocks = (int)std::min<int64_t>(ceil_div64(rows * Cpad, 256), 132 * 32);
    if (t == Half16::FP16) f32_to_split_kernel<true><<<blocks, 256, 0, s>>>(x, y.hi, y.lo, rows, C, Cpad);
    else f32_to_split_kernel<false><<<blocks, 256, 0, s>>>(x, y.hi, y.lo, rows, C, Cpad);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}
int launch_split_to_f32(Split x, float* y, int64_t rows, int C, int Cpad, Half16 t, cudaStream_t s) {
    if (x.l8) {
        f8c_to_f32_kernel<<<(int)std::min<int64_t>(ceil_div64(rows * C, 256), 132 * 32), 256, 0, s>>>(x.hi, x.l8, y, rows, C, Cpad);
        H3D_CHECK_LAUNCH();
        return H3D_OK;
    }
    const int blocks = (int)std::min<int64_t>(ceil_div64(rows * C, 256), 132 * 32);
    if (t == Half16::FP16) split_to_f32_kernel<true><<<blocks, 256, 0, s>>>(x.hi, x.lo, y, rows, C, Cpad);
    else split_to_f32_kernel<false><<<blocks, 256, 0, s>>>(x.hi, x.lo, y, rows, C, Cpad);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

__global__ void copy_channels_kernel(const float* __restrict__ src, float* __restrict__ dst, int64_t rows, int C, int dst_total, int dst_off) {
    const int64_t total = rows * C;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        dst[(i / C) * dst_total + dst_off + c] = src[i];
    }
}
int launch_copy_channels(const float* src, float* dst, int64_t rows, int C, int dst_total, int dst_off, cudaStream_t s) {
    copy_channels_kernel<<<(int)std::min<int64_t>(ceil_div64(rows * C, 256), 132 * 8), 256, 0, s>>>(src, dst, rows, C, dst_total, dst_off);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

// =============================================================================================
// single_obj_scoremap + calc_center_bb + crop scale (utils/general.py:233-328, nets/...:83-85)
//
// Kernel 1 (seg_prob_kernel): per pixel fg = softmax(l)[1] (Eigen form e * (1/sum), SURVEY 9.4),
//   det = round_half_even(fg) == 1  <=>  fg > 0.5, bit-packed with __ballot_sync (bit i of word w of
//   row y <-> pixel x = 32 w + i), and per-image arg-max of fg with first-occurrence tie-break
//   via a 64-bit (value bits, ~index) key reduced with warp shuffles and one atomicMax per block.
// Kernel 2 (mask_grow_kernel): one CTA per image; det / obj bit masks live in shared memory;
//   obj <- det AND dilate21x21(obj), exactly max(H,W)//10 passes (early exit once a pass changes
//   nothing -- the fixed point is idempotent, so the result is identical); then the bounding box,
//   centre, crop size and scale_crop = clip(256 / (1.25 size), 0.25, 5).
// =============================================================================================
struct SegScratch {
    unsigned long long* key;  // [B]
    uint32_t* det;            // [B][H][Ww]
};

__host__ __device__ inline int seg_words(int W) { return (W + 31) >> 5; }

int64_t seg_scratch_bytes(int B, int H, int W) {
    return align_up((int64_t)B * 8, 256) + align_up((int64_t)B * H * seg_words(W) * 4, 256);
}

// UPS = false: `logits` is the full-resolution map [B,H,W,2] (operator entry h3d_seg_postprocess).
// UPS = true (pipeline): `logits` is HandSegNet's low-resolution head output [B,LH,LW,2]; the kernel up-samples it on the fly with exactly
// the operations of resize_bilinear_tf1_kernel<2> (nets/...:166), WRITES the full-resolution hand_scoremap to `up` and classifies the
// values it has in registers - the 0.82 MB / image map is written once and never read back (it was: written, then re-read).
template <bool UPS>
__global__ void __launch_bounds__(256)
seg_prob_kernel(const float2* __restrict__ logits, float2* __restrict__ up, int LH, int LW, float hscale, float wscale, int H, int W,
                int Ww, unsigned long long* __restrict__ key, uint32_t* __restrict__ det) {
    const int b = blockIdx.y;
    const int lane = threadIdx.x & 31;
    const int warps_per_block = blockDim.x >> 5;
    const int words = H * Ww;
    unsigned long long best = 0ull;
    for (int wd = blockIdx.x * warps_per_block + (threadIdx.x >> 5); wd < words; wd += gridDim.x * warps_per_block) {
        const int y = wd / Ww, xw = wd - y * Ww;
        const int x = xw * 32 + lane;
        bool bit = false;
        if (x < W) {
            const int idx = y * W + x;
            float2 l;
            if (UPS) {
                const float in_y = __fmul_rn((float)y, hscale), in_x = __fmul_rn((float)x, wscale);
                const int y0 = (int)floorf(in_y), x0 = (int)floorf(in_x);
                const int y1 = min(y0 + 1, LH - 1), x1 = min(x0 + 1, LW - 1);
                const float ly = __fsub_rn(in_y, (float)y0), lx = __fsub_rn(in_x, (float)x0);
                const float2* r0 = logits + ((int64_t)b * LH + y0) * LW;
                const float2* r1 = logits + ((int64_t)b * LH + y1) * LW;
                const float2 tl = __ldg(r0 + x0), tr = __ldg(r0 + x1), bl = __ldg(r1 + x0), br = __ldg(r1 + x1);
                l.x = lerp_tf(lerp_tf(tl.x, tr.x, lx), lerp_tf(bl.x, br.x, lx), ly);
                l.y = lerp_tf(lerp_tf(tl.y, tr.y, lx), lerp_tf(bl.y, br.y, lx), ly);
                up[(int64_t)b * H * W + idx] = l;
            } else {
                l = __ldg(logits + (int64_t)b * H * W + idx);
            }
            const float m = fmaxf(l.x, l.y);
            const float e0 = expf(__fsub_rn(l.x, m)), e1 = expf(__fsub_rn(l.y, m));
            const float inv = __fdiv_rn(1.0f, __fadd_rn(e0, e1));
            const float fg = __fmul_rn(e1, inv);
            bit = fg > 0.5f;  // == (rint(fg) == 1) for fg in [0,1]
            const unsigned long long k = ((unsigned long long)__float_as_uint(fg) << 32) | (uint32_t)(0xFFFFFFFFu - (uint32_t)idx);
            best = k > best ? k : best;
        }
        const uint32_t word = __ballot_sync(0xFFFFFFFFu, bit);
        if (lane == 0) det[(int64_t)b * words + wd] = word;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long other = __shfl_xor_sync(0xFFFFFFFFu, best, o);
        best = other > best ? other : best;
    }
    __shared__ unsigned long long sbest[32];
    if (lane == 0) sbest[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x < 32) {
        best = threadIdx.x < warps_per_block ? sbest[threadIdx.x] : 0ull;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long other = __shfl_xor_sync(0xFFFFFFFFu, best, o);
            best = other > best ? other : best;
        }
        if (threadIdx.x == 0) atomicMax(key + b, best);
    }
}

constexpr int kGrowThreads = 1024;
constexpr int kMaxMaskWords = 512 * 16;  // H, W <= 512
constexpr int kGrowRows = 8;             // rows per thread in the vertical phase
constexpr int kGrowSeg = 4;              // words per thread in the horizontal phase
constexpr int kGrowPadTop = 10, kGrowPadBot = 10 + kGrowRows - 1;
__host__ __device__ inline int grow_rows_padded(int H) { return (H + kGrowRows - 1) / kGrowRows * kGrowRows; }
// shared memory: det, obj [Hp][Ww] (Hp = H rounded up to 8, padding rows zero) and hor [10 + Hp + 17][Ww] (padding rows zero)
__host__ __device__ inline size_t grow_smem_bytes(int H, int Ww) {
    return (size_t)(2 * grow_rows_padded(H) + kGrowPadTop + grow_rows_padded(H) + kGrowPadBot) * Ww * sizeof(uint32_t);
}

__global__ void __launch_bounds__(kGrowThreads, 1)
mask_grow_kernel(const unsigned long long* __restrict__ key, const uint32_t* __restrict__ det_g, int H, int W, int Ww,
                 int num_passes, uint8_t* __restrict__ hand_mask, int32_t* __restrict__ max_loc, float* __restrict__ center,
                 float* __restrict__ crop_size, float* __restrict__ scale_crop) {
    extern __shared__ uint32_t sm[];
    const int Hp = grow_rows_padded(H);
    uint32_t* det = sm;                                   // [Hp][Ww]
    uint32_t* obj = sm + Hp * Ww;                         // [Hp][Ww]
    uint32_t* hor_p = sm + 2 * Hp * Ww;                   // [10 + Hp + 17][Ww]: row y of the image is row y + 10
    uint32_t* hor = hor_p + kGrowPadTop * Ww;
    __shared__ int s_rmin, s_rmax, s_cmin, s_cmax;
    const int b = blockIdx.x;
    const int words = H * Ww;
    const int tid = threadIdx.x;

    const unsigned long long k = key[b];
    const int seed_idx = (int)(0xFFFFFFFFu - (uint32_t)(k & 0xFFFFFFFFull));
    const int sy = seed_idx / W, sx = seed_idx - sy * W;
    for (int i = tid; i < Hp * Ww; i += kGrowThreads) {
        det[i] = i < words ? det_g[(int64_t)b * words + i] : 0u;
        obj[i] = 0u;
    }
    for (int i = tid; i < (kGrowPadTop + Hp + kGrowPadBot) * Ww; i += kGrowThreads) hor_p[i] = 0u;
    if (tid == 0) {
        s_rmin = 1 << 30; s_rmax = -1; s_cmin = 1 << 30; s_cmax = -1;
        if (max_loc) { max_loc[2 * b] = sy; max_loc[2 * b + 1] = sx; }
    }
    __syncthreads();
    if (tid == 0) obj[sy * Ww + (sx >> 5)] = 1u << (sx & 31);   // one-hot seed (utils/general.py:252-253)
    __syncthreads();

    // One pass = obj <- det AND dilate21x21(obj).  The 21 x 21 box dilation is separable; the SM is instruction-issue bound on it (one
    // CTA per image), so both phases are organised for few instructions per word:
    //  * horizontal (bits): one thread per run of 4 words of a row; the run plus one neighbour word on either side (6 words in registers)
    //    is widened by -+1, -+2, -+4, -+3 pixels (windows 3 -> 7 -> 15 -> 21 pixels: 4 funnel-shift steps instead of 20); the missing
    //    outer neighbours only corrupt the outer 10 bits of the two side words, which the 4 inner words never see;
    //  * vertical (rows) + combine: one thread per (word column, group of 8 rows): the 28 rows [y0-10, y0+17] are read once (zero
    //    padding rows above and below: no bounds checks), the 14 rows common to the eight windows are OR-ed once and the 7 + 7 rows at
    //    either end enter as running prefixes; the result is AND-ed with det, compared with obj and written back (obj is only read in the
    //    horizontal phase).
    // Two block barriers per pass; the second one also carries the "something changed" vote (__syncthreads_or).
    const int segs = (Ww + kGrowSeg - 1) / kGrowSeg;
    const int h_tasks = H * segs;                          // <= 2048: at most two per thread
    int h_base[2], h_x0[2];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
        const int t = tid + q * kGrowThreads;
        const int y = t / segs, sg = t - y * segs;
        h_x0[q] = sg * kGrowSeg;
        h_base[q] = t < h_tasks ? y * Ww + sg * kGrowSeg : -1;
    }
    const int groups = Hp / kGrowRows;
    const int v_tasks = groups * Ww;                       // <= 64 * 16 = 1024: at most one per thread
    const int v_g = tid / Ww, v_xw = tid - v_g * Ww;
    const int v_base = v_g * kGrowRows * Ww + v_xw;        // word of (row y0, column xw); rows advance by Ww words
    for (int pass = 0; pass < num_passes; ++pass) {
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            if (h_base[q] >= 0) {
                const int base = h_base[q], x0 = h_x0[q];
                uint32_t w[kGrowSeg + 2];
#pragma unroll
                for (int i = 0; i < kGrowSeg + 2; ++i) {
                    const int xw = x0 - 1 + i;
                    w[i] = (xw >= 0 && xw < Ww) ? obj[base - 1 + i] : 0u;
                }
#pragma unroll
                for (int step = 0; step < 4; ++step) {
                    const int sft = step == 0 ? 1 : step == 1 ? 2 : step == 2 ? 4 : 3;
                    uint32_t r[kGrowSeg + 2];
#pragma unroll
                    for (int i = 0; i < kGrowSeg + 2; ++i) {
                        const uint32_t lo = i > 0 ? w[i - 1] : 0u, hi = i + 1 < kGrowSeg + 2 ? w[i + 1] : 0u;
                        r[i] = w[i] | __funnelshift_l(lo, w[i], sft) | __funnelshift_r(w[i], hi, sft);
                    }
#pragma unroll
                    for (int i = 0; i < kGrowSeg + 2; ++i) w[i] = r[i];
                }
#pragma unroll
                for (int i = 0; i < kGrowSeg; ++i)
                    if (x0 + i < Ww) hor[base + i] = w[i + 1];      // bits beyond W in the last word are masked by det below
            }
        }
        __syncthreads();
        int changed = 0;
        if (tid < v_tasks) {
            uint32_t v[kGrowRows + 20];
#pragma unroll
            for (int i = 0; i < kGrowRows + 20; ++i) v[i] = hor_p[v_base + i * Ww];   // rows y0 - 10 .. y0 + 17
            uint32_t core = v[kGrowRows - 1];
#pragma unroll
            for (int i = kGrowRows; i <= 20; ++i) core |= v[i];                       // rows common to the windows of y0 .. y0 + 7
            uint32_t lo[kGrowRows], hi[kGrowRows];                                     // lo[k] = v[7-k .. 6], hi[k] = v[21 .. 20+k]; [0] = 0
            lo[0] = 0u; hi[0] = 0u;
#pragma unroll
            for (int kk = 1; kk < kGrowRows; ++kk) { lo[kk] = lo[kk - 1] | v[kGrowRows - 1 - kk]; hi[kk] = hi[kk - 1] | v[20 + kk]; }
#pragma unroll
            for (int j = 0; j < kGrowRows; ++j) {
                const int i = v_base + j * Ww;                                         // padding rows: det = 0 -> obj stays 0
                const uint32_t r = (core | lo[kGrowRows - 1 - j] | hi[j]) & det[i];
                changed |= (r != obj[i]);
                obj[i] = r;
            }
        }
        if (!__syncthreads_or(changed)) break;   // fixed point: remaining passes are no-ops
    }

    // bounding box (utils/general.py:294-300): X = row index, Y = column index
    int rmin = 1 << 30, rmax = -1, cmin = 1 << 30, cmax = -1;
    for (int i = tid; i < words; i += kGrowThreads) {
        const uint32_t v = obj[i];
        if (v) {
            const int y = i / Ww, xw = i - y * Ww;
            rmin = min(rmin, y); rmax = max(rmax, y);
            cmin = min(cmin, xw * 32 + __ffs(v) - 1);
            cmax = max(cmax, xw * 32 + 31 - __clz(v));
        }
    }
    if (rmax >= 0) {
        atomicMin(&s_rmin, rmin); atomicMax(&s_rmax, rmax);
        atomicMin(&s_cmin, cmin); atomicMax(&s_cmax, cmax);
    }
    if (hand_mask) {
        for (int i = tid; i < H * W; i += kGrowThreads) {
            const int y = i / W, x = i - y * W;
            hand_mask[(int64_t)b * H * W + i] = (obj[y * Ww + (x >> 5)] >> (x & 31)) & 1u;
        }
    }
    __syncthreads();
    if (tid == 0) {
        float c0, c1, sz;
        if (s_rmax < 0) {           // empty mask: the reference's written fallbacks (utils/general.py:311-312,319-320)
            c0 = 160.0f; c1 = 160.0f; sz = 100.0f;
        } else {
            const float xmin = (float)s_rmin, xmax = (float)s_rmax, ymin = (float)s_cmin, ymax = (float)s_cmax;
            c0 = __fmul_rn(0.5f, __fadd_rn(xmax, xmin));
            c1 = __fmul_rn(0.5f, __fadd_rn(ymax, ymin));
            sz = fmaxf(__fsub_rn(xmax, xmin), __fsub_rn(ymax, ymin));
        }
        center[2 * b] = c0; center[2 * b + 1] = c1;
        if (crop_size) crop_size[b] = sz;
        const float best = __fmul_rn(sz, 1.25f);                                   // nets/...:84
        scale_crop[b] = fminf(fmaxf(__fdiv_rn(256.0f, best), 0.25f), 5.0f);         // nets/...:85 (size 0 -> inf -> 5)
    }
}

// low != nullptr: fused form for the pipeline - `low` [B,LH,LW,2] is up-sampled to `logits` [B,H,W,2] (written) and classified in one pass
int launch_seg_postprocess(const float* logits, int B, int H, int W, void* scratch, uint8_t* hand_mask, int32_t* max_loc,
                           float* center, float* crop_size, float* scale_crop, cudaStream_t s, int* n_launch, const float* low, int LH,
                           int LW) {
    H3D_REQUIRE(H <= 512 && W <= 512 && H > 0 && W > 0, "seg_postprocess: H, W must be in [1, 512]");
    const int Ww = seg_words(W);
    unsigned long long* key = (unsigned long long*)scratch;
    uint32_t* det = (uint32_t*)((char*)scratch + align_up((int64_t)B * 8, 256));
    H3D_CUDA(cudaMemsetAsync(key, 0, (size_t)B * 8, s));
    const int words = H * Ww;
    // about one resident wave of 256-thread CTAs (132 SMs x 8), split over the images
    dim3 grid(std::max(1, std::min(ceil_div(words, 8), ceil_div(132 * 8, B))), B);
    if (low && !(LH == H && LW == W))
        seg_prob_kernel<true><<<grid, 256, 0, s>>>((const float2*)low, (float2*)const_cast<float*>(logits), LH, LW, (float)LH / (float)H,
                                                   (float)LW / (float)W, H, W, Ww, key, det);
    else
        seg_prob_kernel<false><<<grid, 256, 0, s>>>((const float2*)(low ? low : logits), nullptr, 0, 0, 0.f, 0.f, H, W, Ww, key, det);
    H3D_CHECK_LAUNCH();
    const size_t smem = grow_smem_bytes(H, Ww);    // det, obj, hor (+ zero padding rows)
    static bool attr_set[64] = {};   // per device (one process may drive several GPUs)
    int dev = 0;
    H3D_CUDA(cudaGetDevice(&dev));
    if (!attr_set[dev & 63]) {
        H3D_CUDA(cudaFuncSetAttribute(mask_grow_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)grow_smem_bytes(512, 16)));
        attr_set[dev & 63] = true;
    }
    const int num_passes = std::max(H, W) / (21 / 2);   // utils/general.py:256
    mask_grow_kernel<<<B, kGrowThreads, smem, s>>>(key, det, H, W, Ww, num_passes, hand_mask, max_loc, center, crop_size,
                                                   scale_crop);
    H3D_CHECK_LAUNCH();
    if (n_launch) *n_launch += 2;
    return H3D_OK;
}

// =============================================================================================
// crop_image_from_xy (utils/general.py:163-196) = box arithmetic + tf.image.crop_and_resize
// (bilinear, extrapolation 0; SURVEY 9.9).
// =============================================================================================
struct CropBox { float oy, ox, hs, ws, cy, cx; };
// the box arithmetic of utils/general.py:181-191 and of crop_and_resize_op.cc (per image; every thread evaluates it: ~10 flops on three
// cached scalars cost less than a block barrier at the head of a 20 us kernel)
__device__ __forceinline__ CropBox crop_box(const float* __restrict__ center, const float* __restrict__ scale, int b, int H, int W, int crop) {
    const float hm1 = (float)(H - 1), wm1 = (float)(W - 1);
    const float cs = (float)crop;
    const float css = __fdiv_rn(cs, __ldg(scale + b));               // :182
    const float half = floorf(__fdiv_rn(css, 2.0f));                 // float '//' (:183,185)
    const float y1 = __fsub_rn(__ldg(center + 2 * b), half), y2 = __fadd_rn(y1, css);
    const float x1 = __fsub_rn(__ldg(center + 2 * b + 1), half), x2 = __fadd_rn(x1, css);
    const float y1n = __fdiv_rn(y1, (float)H), y2n = __fdiv_rn(y2, (float)H);   // :187-190 (H, W -- not H-1)
    const float x1n = __fdiv_rn(x1, (float)W), x2n = __fdiv_rn(x2, (float)W);
    CropBox c;
    c.oy = __fmul_rn(y1n, hm1);
    c.ox = __fmul_rn(x1n, wm1);
    c.hs = crop > 1 ? __fdiv_rn(__fmul_rn(__fsub_rn(y2n, y1n), hm1), (float)(crop - 1)) : 0.f;
    c.ws = crop > 1 ? __fdiv_rn(__fmul_rn(__fsub_rn(x2n, x1n), wm1), (float)(crop - 1)) : 0.f;
    c.cy = __fmul_rn(__fmul_rn(0.5f, __fadd_rn(y1n, y2n)), hm1);     // single-row / single-column crops sample the box centre
    c.cx = __fmul_rn(__fmul_rn(0.5f, __fadd_rn(x1n, x2n)), wm1);
    return c;
}

// One thread per output pixel (all C channels, C <= 4); a CTA owns whole output rows of one image (blockIdx.y), so that the 2 input
// rows a row of the crop touches are shared through L1 by its threads; the loop is unrolled by two for loads in flight.
__global__ void __launch_bounds__(256)
crop_image_kernel(const float* __restrict__ image, const float* __restrict__ center, const float* __restrict__ scale,
                  float* __restrict__ out, int B, int H, int W, int C, int crop) {
    const int b = blockIdx.y;
    const float hm1 = (float)(H - 1), wm1 = (float)(W - 1);
    const CropBox bx = crop_box(center, scale, b, H, W, crop);
    const float* img = image + (int64_t)b * H * W * C;
    float* ob = out + (int64_t)b * crop * crop * C;
    const int total = crop * crop;
    const int stride = gridDim.x * blockDim.x;
#pragma unroll 2
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const int y = i / crop, x = i - y * crop;
        const float in_y = crop > 1 ? __fadd_rn(bx.oy, __fmul_rn((float)y, bx.hs)) : bx.cy;
        const float in_x = crop > 1 ? __fadd_rn(bx.ox, __fmul_rn((float)x, bx.ws)) : bx.cx;
        float* dst = ob + (int64_t)i * C;
        const bool valid = !(in_y < 0.f || in_y > hm1) && !(in_x < 0.f || in_x > wm1);
        if (!valid) {
            for (int c = 0; c < C; ++c) dst[c] = 0.f;
            continue;
        }
        const int top = (int)floorf(in_y), bot = (int)ceilf(in_y);
        const int lef = (int)floorf(in_x), rig = (int)ceilf(in_x);
        const float ly = __fsub_rn(in_y, (float)top), lx = __fsub_rn(in_x, (float)lef);
        const float* ptl = img + ((int64_t)top * W + lef) * C;
        const float* ptr = img + ((int64_t)top * W + rig) * C;
        const float* pbl = img + ((int64_t)bot * W + lef) * C;
        const float* pbr = img + ((int64_t)bot * W + rig) * C;
        if (C == 3) {   // the RGB image of the hot path: twelve independent loads in flight, three coalesced stores
            const float tl0 = __ldg(ptl), tl1 = __ldg(ptl + 1), tl2 = __ldg(ptl + 2), tr0 = __ldg(ptr), tr1 = __ldg(ptr + 1), tr2 = __ldg(ptr + 2);
            const float bl0 = __ldg(pbl), bl1 = __ldg(pbl + 1), bl2 = __ldg(pbl + 2), br0 = __ldg(pbr), br1 = __ldg(pbr + 1), br2 = __ldg(pbr + 2);
            dst[0] = lerp_tf(lerp_tf(tl0, tr0, lx), lerp_tf(bl0, br0, lx), ly);
            dst[1] = lerp_tf(lerp_tf(tl1, tr1, lx), lerp_tf(bl1, br1, lx), ly);
            dst[2] = lerp_tf(lerp_tf(tl2, tr2, lx), lerp_tf(bl2, br2, lx), ly);
        } else {
            for (int c = 0; c < C; ++c)
                dst[c] = lerp_tf(lerp_tf(__ldg(ptl + c), __ldg(ptr + c), lx), lerp_tf(__ldg(pbl + c), __ldg(pbr + c), lx), ly);
        }
    }
}

int launch_crop_image(const float* image, const float* center, const float* scale, float* out, int B, int H, int W, int C,
                      int crop, cudaStream_t s) {
    const int total = crop * crop;
    // about one resident wave: 132 SMs x 8 CTAs of 256 threads, split over the images (at least 1, at most one CTA per 256 pixels)
    const int per_image = std::max(1, std::min(ceil_div(total, 256), ceil_div(132 * 8, std::max(1, B))));
    crop_image_kernel<<<dim3((unsigned)per_image, B), 256, 0, s>>>(image, center, scale, out, B, H, W, C, crop);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

// =============================================================================================
// detect_keypoints (utils/general.py:331-344), batched on device.  Thread (p, c) streams pixels
// p, p+P, ... of channel c: consecutive threads read consecutive floats (NHWC), keys are reduced in
// shared memory and merged with one 64-bit atomicMax per (block, channel).
// =============================================================================================
__device__ __forceinline__ uint32_t float_orderable(float v) {
    const uint32_t u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

int64_t argmax_scratch_bytes(int B, int C) { return align_up((int64_t)B * C * 8, 256); }

__global__ void heatmap_argmax_kernel(const float* __restrict__ sm, int HW, int C, int P, unsigned long long* __restrict__ key) {
    extern __shared__ unsigned long long skey[];   // [P][C]
    const int b = blockIdx.y;
    const int t = threadIdx.x;
    const int p_sub = t / C, c = t - p_sub * C;
    unsigned long long best = 0ull;
    if (p_sub < P) {
        const float* base = sm + (int64_t)b * HW * C;
        for (int p = blockIdx.x * P + p_sub; p < HW; p += gridDim.x * P) {
            const float v = __ldg(base + (int64_t)p * C + c);
            const unsigned long long k = ((unsigned long long)float_orderable(v) << 32) | (uint32_t)(0xFFFFFFFFu - (uint32_t)p);
            best = k > best ? k : best;
        }
        skey[p_sub * C + c] = best;
    }
    __syncthreads();
    if (t < C) {
        unsigned long long m = 0ull;
        for (int q = 0; q < P; ++q) { const unsigned long long k = skey[q * C + t]; m = k > m ? k : m; }
        atomicMax(key + (int64_t)b * C + t, m);
    }
}

__global__ void argmax_decode_kernel(const unsigned long long* __restrict__ key, int n, int W, int32_t* __restrict__ uv) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const int idx = (int)(0xFFFFFFFFu - (uint32_t)(key[i] & 0xFFFFFFFFull));
        uv[2 * i] = idx / W;       // v (row)
        uv[2 * i + 1] = idx % W;   // u (col)
    }
}

int launch_detect_keypoints(const float* sm, int B, int H, int W, int C, void* scratch, int32_t* uv, cudaStream_t s,
                            int* n_launch) {
    H3D_REQUIRE(C >= 1 && C <= 256, "detect_keypoints: C must be in [1,256]");
    unsigned long long* key = (unsigned long long*)scratch;
    H3D_CUDA(cudaMemsetAsync(key, 0, (size_t)B * C * 8, s));
    const int P = std::max(1, 256 / C);
    const int threads = P * C;
    const int HW = H * W;
    dim3 grid(std::max(1, std::min(ceil_div(HW, P * 16), 64)), B);
    heatmap_argmax_kernel<<<grid, threads, (size_t)P * C * 8, s>>>(sm, HW, C, P, key);
    H3D_CHECK_LAUNCH();
    argmax_decode_kernel<<<ceil_div(B * C, 256), 256, 0, s>>>(key, B * C, W, uv);
    H3D_CHECK_LAUNCH();
    if (n_launch) *n_launch += 2;
    return H3D_OK;
}

// =============================================================================================
// _get_rot_mat + _flip_right_hand + batched matmul (nets/ColorHandPose3DNetwork.py:239-247,311-384)
// =============================================================================================
__global__ void rotate_canonical_kernel(const float* __restrict__ can, const float* __restrict__ uxyz,
                                        const float* __restrict__ hand_side, int B, float* __restrict__ rot, float* __restrict__ out) {
    const int b = blockIdx.x;
    __shared__ float R[9];
    if (threadIdx.x == 0) {
        rodrigues_rot_mat(uxyz[3 * b], uxyz[3 * b + 1], uxyz[3 * b + 2], R);
        if (rot)
            for (int i = 0; i < 9; ++i) rot[9 * b + i] = R[i];
    }
    __syncthreads();
    const bool right = hand_side[2 * b + 1] > hand_side[2 * b];   // argmax(hand_side,1)==1 (ties -> index 0)
    for (int i = threadIdx.x; i < 63; i += blockDim.x) out[63 * b + i] = rotate_canonical_point(can + 63 * b, R, i, right);
}

// =============================================================================================
// Fused x8 up-sampling + detect_keypoints: writes the TF1-legacy bilinear up-sampled score map (nets/...:96-97) and
// reduces its per-channel first-occurrence arg-max (utils/general.py:331-344) in the same pass, so the 5.5 MB/image map
// is written once and never re-read.  Thread (p_sub, c) produces pixels p_sub, p_sub + P, ... of channel c: the C threads
// of a pixel write C consecutive floats.  Values are computed exactly as resize_bilinear_tf1_kernel computes them.
// =============================================================================================
template <int C>
__global__ void resize_argmax_kernel(const float* __restrict__ x, float* __restrict__ y, int H, int W, int oh, int ow, float hscale,
                                     float wscale, int P, unsigned long long* __restrict__ key) {
    extern __shared__ unsigned long long skey[];   // [P][C]
    const int b = blockIdx.y;
    const int t = threadIdx.x;
    const int p_sub = t / C, c = t - p_sub * C;
    const int HW = oh * ow;
    unsigned long long best = 0ull;
    if (p_sub < P) {
        const float* xb = x + (int64_t)b * H * W * C;
        float* yb = y + (int64_t)b * HW * C;
        for (int p = blockIdx.x * P + p_sub; p < HW; p += gridDim.x * P) {
            const int oy = p / ow, ox = p - oy * ow;
            const float in_y = __fmul_rn((float)oy, hscale), in_x = __fmul_rn((float)ox, wscale);
            const int y0 = (int)floorf(in_y), x0 = (int)floorf(in_x);
            const int y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
            const float ly = __fsub_rn(in_y, (float)y0), lx = __fsub_rn(in_x, (float)x0);
            const float tl = __ldg(xb + (y0 * W + x0) * C + c), tr = __ldg(xb + (y0 * W + x1) * C + c);
            const float bl = __ldg(xb + (y1 * W + x0) * C + c), br = __ldg(xb + (y1 * W + x1) * C + c);
            const float v = lerp_tf(lerp_tf(tl, tr, lx), lerp_tf(bl, br, lx), ly);
            yb[(int64_t)p * C + c] = v;
            const unsigned long long k = ((unsigned long long)float_orderable(v) << 32) | (uint32_t)(0xFFFFFFFFu - (uint32_t)p);
            best = k > best ? k : best;
        }
        skey[p_sub * C + c] = best;
    }
    __syncthreads();
    if (t < C) {
        unsigned long long m = 0ull;
        for (int q = 0; q < P; ++q) { const unsigned long long k = skey[q * C + t]; m = k > m ? k : m; }
        atomicMax(key + (int64_t)b * C + t, m);
    }
}

// Power-of-two integer up-sampling (the x8 of nets/ColorHandPose3DNetwork.py:96-97) restructured for instruction count: with scale
// 1/s exact in fp32, the s output rows oy = s y0 .. s y0 + s - 1 share the input rows (y0, y1) and therefore the horizontal
// interpolants top(ox) / bot(ox): one CTA per (image, y0) stages the two input rows in shared memory, every thread owns ONE 16-byte
// output column group (4 consecutive floats of the flattened (ox, c) row; the channel pattern of a group repeats every 4 pixels =
// 84 floats, so a thread's four channels are fixed), computes top / bot once and emits s rows with one vertical lerp + one arg-max
// update per value and 16-byte stores.  Values are computed by exactly the operations of resize_bilinear_tf1_kernel.
template <int C>
__global__ void resize_argmax_pow2_kernel(const float* __restrict__ x, float* __restrict__ y, int H, int W, int s_log2, float hscale,
                                          float wscale, unsigned long long* __restrict__ key) {
    static_assert((4 * C) % 4 == 0, "");
    constexpr int G4 = C;                        // float4 groups per 4 output pixels (4 C floats)
    extern __shared__ unsigned long long sdyn[];
    float* rows = reinterpret_cast<float*>(sdyn);                         // [2][W * C]
    unsigned long long* skey = sdyn + (2 * W * C + 1) / 2;                // [C][slots]
    const int sfac = 1 << s_log2;
    const int ow = W << s_log2;
    const int b = blockIdx.y, y0 = blockIdx.x;
    const int y1 = min(y0 + 1, H - 1);
    const int t = threadIdx.x;
    const int j = t % G4, gsub = t / G4, gstep = blockDim.x / G4;          // float4 index inside the 4-pixel group, pixel-group lane
    const float* xb = x + (int64_t)b * H * W * C;
    for (int i = t; i < W * C; i += blockDim.x) { rows[i] = __ldg(xb + (int64_t)y0 * W * C + i); rows[W * C + i] = __ldg(xb + (int64_t)y1 * W * C + i); }
    __syncthreads();
    int pofs[4], cc[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { pofs[i] = (4 * j + i) / C; cc[i] = (4 * j + i) % C; }
    float bv[4] = {0.f, 0.f, 0.f, 0.f};
    int bp[4] = {0x7fffffff, 0x7fffffff, 0x7fffffff, 0x7fffffff};
    bool have[4] = {false, false, false, false};
    const int groups = ow >> 2;                   // 4-pixel groups per output row
    float* yb = y + (int64_t)b * (int64_t)(H << s_log2) * ow * C;
    if (gsub < gstep) {
        for (int g = gsub; g < groups; g += gstep) {
            float top[4], bot[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int ox = 4 * g + pofs[i];
                const float in_x = __fmul_rn((float)ox, wscale);
                const int x0 = (int)floorf(in_x), x1 = min(x0 + 1, W - 1);
                const float lx = __fsub_rn(in_x, (float)x0);
                top[i] = lerp_tf(rows[x0 * C + cc[i]], rows[x1 * C + cc[i]], lx);
                bot[i] = lerp_tf(rows[W * C + x0 * C + cc[i]], rows[W * C + x1 * C + cc[i]], lx);
            }
            for (int r = 0; r < sfac; ++r) {
                const int oy = (y0 << s_log2) + r;
                const float in_y = __fmul_rn((float)oy, hscale);
                const float ly = __fsub_rn(in_y, (float)y0);            // floor(in_y) == y0 exactly for a power-of-two scale
                float o[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    o[i] = lerp_tf(top[i], bot[i], ly);
                    const int pidx = oy * ow + 4 * g + pofs[i];
                    if (!have[i] || o[i] > bv[i] || (o[i] == bv[i] && pidx < bp[i])) { bv[i] = o[i]; bp[i] = pidx; have[i] = true; }
                }
                *reinterpret_cast<float4*>(yb + ((int64_t)oy * ow + 4 * g) * C + 4 * j) = make_float4(o[0], o[1], o[2], o[3]);
            }
        }
    }
    // per-channel reduction: slot (gsub, j-slot) -> skey[c][...]; every channel occurs in exactly 4 (j, i) pairs
    const int slots = 4 * gstep;
    for (int i = t; i < C * slots; i += blockDim.x) skey[i] = 0ull;
    __syncthreads();
    if (gsub < gstep) {
#pragma unroll
        for (int i = 0; i < 4; ++i)
            if (have[i]) {
                const unsigned long long k = ((unsigned long long)float_orderable(bv[i]) << 32) | (uint32_t)(0xFFFFFFFFu - (uint32_t)bp[i]);
                skey[cc[i] * slots + gsub * 4 + pofs[i]] = k;            // (gsub, pixel offset) is unique per channel
            }
    }
    __syncthreads();
    if (t < C) {
        unsigned long long m = 0ull;
        for (int q = 0; q < slots; ++q) { const unsigned long long k = skey[t * slots + q]; m = k > m ? k : m; }
        atomicMax(key + (int64_t)b * C + t, m);
    }
}

int launch_resize_argmax21(const float* x, float* y, int B, int H, int W, int oh, int ow, void* scratch, int32_t* uv, cudaStream_t s,
                           int* n_launch) {
    constexpr int C = 21;
    unsigned long long* key = (unsigned long long*)scratch;
    H3D_CUDA(cudaMemsetAsync(key, 0, (size_t)B * C * 8, s));
    // integer power-of-two up-sampling in both directions (x8 on the hot path): row-group kernel
    if (oh % H == 0 && ow % W == 0 && oh / H == ow / W && ((oh / H) & (oh / H - 1)) == 0 && oh / H >= 2 && (ow % 4) == 0 &&
        (((uintptr_t)y) & 15) == 0 && (int64_t)W * C * 8 + 4 * 16 * C * 8 <= 48 * 1024) {
        int sl = 0;
        while ((1 << sl) < oh / H) ++sl;
        const int gstep = 16, threads = C * gstep;                        // 336 threads: 21 float4 columns x 16 pixel-group lanes
        const size_t smem = (size_t)((2 * W * C + 1) / 2) * 8 + (size_t)C * 4 * gstep * 8;
        resize_argmax_pow2_kernel<C><<<dim3(H, B), threads, smem, s>>>(x, y, H, W, sl, (float)H / (float)oh, (float)W / (float)ow, key);
        H3D_CHECK_LAUNCH();
        argmax_decode_kernel<<<ceil_div(B * C, 256), 256, 0, s>>>(key, B * C, ow, uv);
        H3D_CHECK_LAUNCH();
        if (n_launch) *n_launch += 2;
        return H3D_OK;
    }
    const int P = 256 / C;
    dim3 grid(std::max(1, std::min(ceil_div(oh * ow, P * 8), 4 * 132 / std::max(1, std::min(B, 4)))), B);
    resize_argmax_kernel<C><<<grid, P * C, (size_t)P * C * 8, s>>>(x, y, H, W, oh, ow, (float)H / (float)oh, (float)W / (float)ow, P, key);
    H3D_CHECK_LAUNCH();
    argmax_decode_kernel<<<ceil_div(B * C, 256), 256, 0, s>>>(key, B * C, ow, uv);
    H3D_CHECK_LAUNCH();
    if (n_launch) *n_launch += 2;
    return H3D_OK;
}

// =============================================================================================
// On-device decode of the readers' fixed-length binary records (SURVEY.md 8(f) row 2):
//   RHD (data/BinaryDbReader.py:103-208, create_binary_db.py:44-87): 42x3 f32 xyz | 42x2 f32 uv | 9 f32 K | 2 B pad |
//        320x320x3 u8 RGB | 320x320 u8 part mask | 42 u8 visibility                    = 410 520 B
//   STB (data/BinaryDbReaderSTB.py:99-185): 21x3 f32 xyz | 21x3 f32 (u, v, valid) | 480x640x3 u8 RGB = 922 104 B
// The float header is copied as is; the image becomes fp32 `u8 / 255 - 0.5` (two fp32 ops, as the readers do), optionally
// sub-sampled by `step` (eval_full.py:50 resizes 480x640 -> 240x320, which TF1's legacy bilinear turns into "every 2nd pixel").
// =============================================================================================
__global__ void decode_records_kernel(const uint8_t* __restrict__ rec, int64_t record_bytes, int header_floats, int64_t image_off,
                                      int H, int W, int step, int64_t mask_off, int tail_bytes, float* __restrict__ header,
                                      float* __restrict__ image, uint8_t* __restrict__ mask, uint8_t* __restrict__ tail, int B) {
    const int Ho = H / step, Wo = W / step;
    const int64_t per_img = (int64_t)Ho * Wo * 3;
    const int64_t total = (int64_t)B * per_img;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int b = (int)(i / per_img);
        const int64_t r = i - (int64_t)b * per_img;
        const int c = (int)(r % 3), x = (int)((r / 3) % Wo), y = (int)(r / (3 * (int64_t)Wo));
        const uint8_t v = rec[(int64_t)b * record_bytes + image_off + ((int64_t)(y * step) * W + x * step) * 3 + c];
        image[i] = __fsub_rn(__fdiv_rn((float)v, 255.0f), 0.5f);
    }
    const int64_t gtid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, gstride = (int64_t)gridDim.x * blockDim.x;
    if (header) {
        for (int64_t i = gtid; i < (int64_t)B * header_floats; i += gstride) {
            const int b = (int)(i / header_floats), j = (int)(i - (int64_t)b * header_floats);
            const uint8_t* p = rec + (int64_t)b * record_bytes + 4 * j;       // records start 4-byte aligned (both sizes are multiples of 4)
            uint32_t u = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
            header[i] = __uint_as_float(u);
        }
    }
    if (mask && mask_off >= 0) {
        const int64_t n = (int64_t)H * W;
        for (int64_t i = gtid; i < (int64_t)B * n; i += gstride) {
            const int b = (int)(i / n);
            mask[i] = rec[(int64_t)b * record_bytes + mask_off + (i - (int64_t)b * n)];
        }
    }
    if (tail && tail_bytes > 0) {
        for (int64_t i = gtid; i < (int64_t)B * tail_bytes; i += gstride) {
            const int b = (int)(i / tail_bytes);
            tail[i] = rec[(int64_t)b * record_bytes + record_bytes - tail_bytes + (i - (int64_t)b * tail_bytes)];
        }
    }
}

int launch_decode_records(const uint8_t* rec, int64_t record_bytes, int header_floats, int64_t image_off, int H, int W, int step,
                          int64_t mask_off, int tail_bytes, float* header, float* image, uint8_t* mask, uint8_t* tail, int B,
                          cudaStream_t s) {
    const int64_t total = (int64_t)B * (H / step) * (W / step) * 3;
    decode_records_kernel<<<(int)std::min<int64_t>(ceil_div64(total, 256), 132 * 16), 256, 0, s>>>(
        rec, record_bytes, header_floats, image_off, H, W, step, mask_off, tail_bytes, header, image, mask, tail, B);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

// =============================================================================================
// EvalUtil.feed (utils/general.py:531-549), batched: euclidean distance per key-point, -1 where not visible.
// =============================================================================================
__global__ void eval_dist_kernel(const float* __restrict__ gt, const uint8_t* __restrict__ vis, const float* __restrict__ pred,
                                 int n, int D, float* __restrict__ dist) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float acc = 0.f;
    for (int d = 0; d < D; ++d) {
        const float df = __fsub_rn(gt[(int64_t)i * D + d], pred[(int64_t)i * D + d]);
        acc = __fadd_rn(acc, __fmul_rn(df, df));
    }
    dist[i] = vis[i] ? sqrtf(acc) : -1.0f;
}

int launch_eval_dist(const float* gt, const uint8_t* vis, const float* pred, int n, int D, float* dist, cudaStream_t s) {
    eval_dist_kernel<<<ceil_div(n, 256), 256, 0, s>>>(gt, vis, pred, n, D, dist);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

// =============================================================================================
// Fused record pack + all-gather over NVLink peer memory (SURVEY.md 8(e) "fusion target").
// Every rank owns a symmetric gather buffer [2 parities][world*B][108] that all peers have mapped.  One CTA packs this
// rank's 432-byte per-image records (coord3d 63 f32 | key-points 42 i32 | center 2 | scale 1) and stores them straight
// into slot `rank` of EVERY peer's buffer (plain st.global on peer-mapped addresses, or one multimem.st on the NVSwitch
// multicast address when available), fences at system scope, raises flag[rank] = epoch in every peer's signal pad and
// then waits until all peers have raised theirs here: when the kernel ends the local buffer holds the full gather.
// No NCCL launch, no separate pack kernel, one kernel on the critical path (payload is latency-bound: 13.8 KB per rank).
// =============================================================================================
__device__ __forceinline__ void st_release_sys_u32(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

__global__ void __launch_bounds__(1024, 1)
gather_records_p2p_kernel(const float* __restrict__ coord3d, const int32_t* __restrict__ uv, const float* __restrict__ center,
                          const float* __restrict__ scale, int B, const uint64_t* __restrict__ peer_buffers,
                          const uint64_t* __restrict__ peer_signals, uint64_t multicast_ptr, int rank, int world, uint32_t epoch,
                          int64_t parity_stride_floats, int64_t slot_floats, int* __restrict__ err_flag) {
    const int n = B * 108;
    // rank r's records live at slot r * slot_floats (slot_floats = max_batch * 108): ranks with different B never overlap
    const int64_t base = (int64_t)(epoch & 1u) * parity_stride_floats + (int64_t)rank * slot_floats;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int b = i / 108, j = i - b * 108;
        float v;
        if (j < 63) v = coord3d[b * 63 + j];
        else if (j < 105) v = __int_as_float(uv[b * 42 + (j - 63)]);
        else if (j < 107) v = center[b * 2 + (j - 105)];
        else v = scale[b];
        if (multicast_ptr) {
            asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" ::"l"(reinterpret_cast<float*>(multicast_ptr) + base + i), "f"(v) : "memory");
        } else {
            for (int r = 0; r < world; ++r) reinterpret_cast<float*>(peer_buffers[r])[base + i] = v;   // peer-mapped NVLink stores
        }
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x < world) {
        const int r = threadIdx.x;
        st_release_sys_u32(reinterpret_cast<uint32_t*>(peer_signals[r]) + rank, epoch);          // "rank's records have landed at r"
        const uint32_t* mine = reinterpret_cast<const uint32_t*>(peer_signals[rank]) + r;
        const long long t0 = clock64();
        while ((int32_t)(ld_acquire_sys_u32(mine) - epoch) < 0) {                                 // wait for peer r's records
            if (clock64() - t0 > 20000000000ll) { if (err_flag) atomicExch_system(err_flag, 100 + r); break; }   // ~10 s: peer r never signalled
        }
    }
    __syncthreads();
}

int launch_gather_records_p2p(const float* coord3d, const int32_t* uv, const float* center, const float* scale, int B,
                              const uint64_t* peer_buffers, const uint64_t* peer_signals, uint64_t multicast_ptr, int rank, int world,
                              uint32_t epoch, int64_t parity_stride_floats, int max_batch, int* err_flag, cudaStream_t s) {
    H3D_REQUIRE(world >= 1 && world <= 64 && rank >= 0 && rank < world && B > 0 && B <= max_batch, "gather_records_p2p: bad geometry");
    gather_records_p2p_kernel<<<1, 1024, 0, s>>>(coord3d, uv, center, scale, B, peer_buffers, peer_signals, multicast_ptr, rank, world,
                                                 epoch, parity_stride_floats, (int64_t)max_batch * 108, err_flag);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

// =============================================================================================
// bone_rel_trafo_inv (utils/relative_trafo.py:243-295): forward kinematics over the 21-node hand chain.
// One thread per (sample, chain): the root key-point and the 5 fingers are independent chains of rigid
// transforms T <- Trans_z(-len) RotX(-ax) RotY(-ay) T; the key-point is inv(T) [0,0,0,1]^T = -R^T t.
// =============================================================================================
__global__ void bone_rel_trafo_inv_kernel(const float* __restrict__ rel, float* __restrict__ xyz, int B) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= B * 6) return;
    const int b = idx / 6, c = idx - b * 6;
    float R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, t[3] = {0, 0, 0};
    const int n = c == 0 ? 1 : 4;
    for (int i = 0; i < n; ++i) {
        const int bone = c == 0 ? 0 : 4 * c - i;        // kinematic_chain_list: 4,3,2,1 | 8,7,6,5 | ...
        const float* r = rel + ((int64_t)b * 21 + bone) * 3;
        const float len = r[0], ax = -r[1], ay = -r[2];
        const float cx = cosf(ax), sx = sinf(ax), cy = cosf(ay), sy = sinf(ay);
        // M = RotX(ax) * RotY(ay)
        const float M[9] = {cy, 0.f, sy, sx * sy, cx, -sx * cy, -cx * sy, sx, cx * cy};
        float Rn[9], tn[3];
#pragma unroll
        for (int i2 = 0; i2 < 3; ++i2) {
#pragma unroll
            for (int j = 0; j < 3; ++j) Rn[3 * i2 + j] = M[3 * i2] * R[j] + M[3 * i2 + 1] * R[3 + j] + M[3 * i2 + 2] * R[6 + j];
            tn[i2] = M[3 * i2] * t[0] + M[3 * i2 + 1] * t[1] + M[3 * i2 + 2] * t[2];
        }
        tn[2] -= len;
#pragma unroll
        for (int j = 0; j < 9; ++j) R[j] = Rn[j];
#pragma unroll
        for (int j = 0; j < 3; ++j) t[j] = tn[j];
        float* o = xyz + ((int64_t)b * 21 + bone) * 3;
#pragma unroll
        for (int j = 0; j < 3; ++j) o[j] = -(R[j] * t[0] + R[3 + j] * t[1] + R[6 + j] * t[2]);
    }
}

int launch_bone_rel_trafo_inv(const float* rel, float* xyz, int B, cudaStream_t s) {
    bone_rel_trafo_inv_kernel<<<ceil_div(B * 6, 128), 128, 0, s>>>(rel, xyz, B);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

int launch_rotate_canonical(const float* coord_can, const float* uxyz, const float* hand_side, int B, float* rot, float* out,
                            cudaStream_t s) {
    rotate_canonical_kernel<<<B, 64, 0, s>>>(coord_can, uxyz, hand_side, B, rot, out);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

// =============================================================================================
// Record pack alone (single-GPU serving path; the multi-GPU path packs inside gather_records_p2p_kernel):
// [B,108] = coord3d 63 f32 | key-points 42 i32 (bit-cast) | center 2 | scale 1.
// =============================================================================================
__global__ void pack_records_kernel(const float* __restrict__ coord3d, const int32_t* __restrict__ uv, const float* __restrict__ center,
                                    const float* __restrict__ scale, int B, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * 108) return;
    const int b = i / 108, j = i - b * 108;
    float v;
    if (j < 63) v = coord3d[b * 63 + j];
    else if (j < 105) v = __int_as_float(uv[b * 42 + (j - 63)]);
    else if (j < 107) v = center[b * 2 + (j - 105)];
    else v = scale[b];
    out[i] = v;
}
int launch_pack_records(const float* coord3d, const int32_t* uv, const float* center, const float* scale, int B, float* out, cudaStream_t s) {
    pack_records_kernel<<<ceil_div(B * 108, 256), 256, 0, s>>>(coord3d, uv, center, scale, B, out);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

// =============================================================================================
// calc_center_bb (utils/general.py:271-328) on an arbitrary mask: one CTA per image reduces the bounding box of the pixels
// with int(mask) == 1 (X = row index, Y = column index as in the reference), then centre = 0.5 (max + min), crop size =
// max extent; an empty mask gives the reference's written fall-backs (centre 160, size 100) and bb = (+inf, -inf).
// =============================================================================================
__global__ void mask_bbox_kernel(const float* __restrict__ mask, int H, int W, float* __restrict__ center, float* __restrict__ bb,
                                 float* __restrict__ crop_size) {
    __shared__ int s_rmin, s_rmax, s_cmin, s_cmax;
    const int b = blockIdx.x;
    if (threadIdx.x == 0) { s_rmin = 1 << 30; s_rmax = -1; s_cmin = 1 << 30; s_cmax = -1; }
    __syncthreads();
    int rmin = 1 << 30, rmax = -1, cmin = 1 << 30, cmax = -1;
    const float* m = mask + (int64_t)b * H * W;
    for (int i = threadIdx.x; i < H * W; i += blockDim.x) {
        if ((int)__ldg(m + i) == 1) {     // tf.cast(mask, tf.int32) == 1 (:274-275)
            const int y = i / W, x = i - y * W;
            rmin = min(rmin, y); rmax = max(rmax, y); cmin = min(cmin, x); cmax = max(cmax, x);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        rmin = min(rmin, __shfl_xor_sync(0xFFFFFFFFu, rmin, o)); rmax = max(rmax, __shfl_xor_sync(0xFFFFFFFFu, rmax, o));
        cmin = min(cmin, __shfl_xor_sync(0xFFFFFFFFu, cmin, o)); cmax = max(cmax, __shfl_xor_sync(0xFFFFFFFFu, cmax, o));
    }
    if ((threadIdx.x & 31) == 0 && rmax >= 0) {
        atomicMin(&s_rmin, rmin); atomicMax(&s_rmax, rmax); atomicMin(&s_cmin, cmin); atomicMax(&s_cmax, cmax);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const float inf = __int_as_float(0x7f800000);
        float c0 = 160.0f, c1 = 160.0f, sz = 100.0f, xmin = inf, xmax = -inf, ymin = inf, ymax = -inf;
        if (s_rmax >= 0) {
            xmin = (float)s_rmin; xmax = (float)s_rmax; ymin = (float)s_cmin; ymax = (float)s_cmax;
            c0 = __fmul_rn(0.5f, __fadd_rn(xmax, xmin));
            c1 = __fmul_rn(0.5f, __fadd_rn(ymax, ymin));
            sz = fmaxf(__fsub_rn(xmax, xmin), __fsub_rn(ymax, ymin));
        }
        center[2 * b] = c0; center[2 * b + 1] = c1;
        if (bb) { bb[4 * b] = xmin; bb[4 * b + 1] = xmax; bb[4 * b + 2] = ymin; bb[4 * b + 3] = ymax; }   // [[x_min, x_max], [y_min, y_max]] (:303)
        if (crop_size) crop_size[b] = sz;
    }
}
int launch_mask_bbox(const float* mask, int B, int H, int W, float* center, float* bb, float* crop_size, cudaStream_t s) {
    mask_bbox_kernel<<<B, 512, 0, s>>>(mask, H, W, center, bb, crop_size);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

// NetworkOps.leaky_relu (utils/general.py:31-33): tf.maximum(x, 0.01 x)
__global__ void leaky_relu_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t n) {
    const int64_t n4 = n >> 2;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
        float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
        v.x = fmaxf(v.x, __fmul_rn(kNegSlope, v.x)); v.y = fmaxf(v.y, __fmul_rn(kNegSlope, v.y));
        v.z = fmaxf(v.z, __fmul_rn(kNegSlope, v.z)); v.w = fmaxf(v.w, __fmul_rn(kNegSlope, v.w));
        reinterpret_cast<float4*>(y)[i] = v;
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
        const int64_t i = (n4 << 2) + threadIdx.x;
        y[i] = fmaxf(x[i], __fmul_rn(kNegSlope, x[i]));
    }
}
int launch_leaky_relu(const float* x, float* y, int64_t n, cudaStream_t s) {
    H3D_REQUIRE((((uintptr_t)x | (uintptr_t)y) & 15) == 0, "leaky_relu: pointers must be 16-byte aligned");
    leaky_relu_kernel<<<(int)std::max<int64_t>(1, std::min<int64_t>(ceil_div64(n / 4 + 1, 256), 132 * 16)), 256, 0, s>>>(x, y, n);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

// _flip_right_hand (nets/ColorHandPose3DNetwork.py:336-361): z -> -z where cond_right[b] != 0
__global__ void flip_right_hand_kernel(const float* __restrict__ xyz, const uint8_t* __restrict__ cond_right, int B, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * 63) return;
    const int b = i / 63, j = (i - b * 63) % 3;
    const float v = xyz[i];
    out[i] = (j == 2 && cond_right[b]) ? -v : v;
}
int launch_flip_right_hand(const float* xyz, const uint8_t* cond_right, int B, float* out, cudaStream_t s) {
    flip_right_hand_kernel<<<ceil_div(B * 63, 256), 256, 0, s>>>(xyz, cond_right, B, out);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

}  // namespace h3d

// Activation storage formats of the tensor-core path ("split" planes) and the scalar conversions every producer uses.
//
//   2-plane 16-bit split (bf16x3 / fp16x3):  x ~= hi + lo,  hi = rn16(x), lo = rn16(x - hi)
//   fp16 + fp8 correction planes (fp16_f8c): x ~= h16 * 2^-5 + l8 * 2^-10, and a coarse copy h8 * 2^2 for the weight-residual term
//        h16 = fp16(x * 2^5)                     (11 significant bits: the main tensor-core pass; saturates at |x| = 2047)
//        l8  = e4m3((x - h16 * 2^-5) * 2^10)     (residual, <= 2^-12 |x|  ->  covers |x| up to 1792)
//        h8  = e4m3(x * 2^-2)                    (x itself at 4 bits, same range; multiplies the fp8 weight residual)
//   Weights: wh16 = fp16(w 2^(5+b)), wh8 = e4m3(w 2^b), wl8 = e4m3((w - wh16 2^-(5+b)) 2^(12+b)).  The three products
//   h16*wh16, l8*wh8 and h8*wl8 then all carry the same factor 2^(10+b) and share ONE fp32 accumulator; the epilogue
//   multiplies by 2^-(10+b) (exact).
//   Range: the activation scales are fixed, so the mode is fp32 grade (scale-relative error <= 1e-5, 4.4e-6 measured on an H100
//   80GB HBM3 at 400 W) only for activations of 2^-2 .. 2^6 times unit scale and layers whose largest |w| is >= ~2.5e-3 (b is per
//   layer and clamped to [-20, 20]); below, the e4m3 residual underflows and the error grows towards plain fp16's; |x| >= 2047
//   saturates the main plane.  Nothing reports either (DESIGN.md section 6.1).
//
//   fp16 weight planes (fp16x3, fp16): every output channel co is packed pre-scaled by 2^s(co), chosen so that
//   max_k |w[k, co]| 2^s lies in [2^13, 2^14) (s = 0 for an all-zero column).  fp16's normal range ends at 2^-14, so without the
//   shift the lo plane of every |w| below ~0.125 (and the hi plane of every |w| below 2^-14) would be subnormal and lose bits.
//   The epilogue multiplies the fp32 accumulator by 2^-s(co) (exact).  bf16 planes have fp32's exponent range and no shift.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <math.h>
#include <stdint.h>

namespace h3d {

// s(co) of the fp16 weight planes from max_k |w[k, co]|; identical on the host packer and the device packer
__host__ __device__ __forceinline__ int fp16_w_shift(float colmax) {
    if (!(colmax > 0.f)) return 0;
    int e;
    frexpf(colmax, &e);   // colmax = m 2^e, m in [0.5, 1)
    const int s = 14 - e;
    return s < -126 ? -126 : (s > 126 ? 126 : s);
}

constexpr float kF8XLoScale = 1024.0f;    // 2^10
constexpr float kF8XHiScale = 0.25f;      // 2^-2
constexpr float kF8XMainScale = 32.0f;    // 2^5
constexpr int kF8XLoShift = 10, kF8XHiShift = -2, kF8XMainShift = 5;

__host__ __device__ __forceinline__ uint8_t f32_to_e4m3(float v) {
    return (uint8_t)__nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E4M3);
}
__host__ __device__ __forceinline__ float e4m3_to_f32(uint8_t v) {
    __half_raw h = __nv_cvt_fp8_to_halfraw((__nv_fp8_storage_t)v, __NV_E4M3);
    return __half2float(*reinterpret_cast<__half*>(&h));
}

struct F8cPlanes { uint16_t h16; uint8_t l8, h8; };
__device__ __forceinline__ F8cPlanes f32_to_f8c(float x) {
    F8cPlanes p;
    const __half h = __float2half_rn(fminf(fmaxf(x * kF8XMainScale, -65504.f), 65504.f));
    p.h16 = __half_as_ushort(h);
    p.l8 = f32_to_e4m3((x - __half2float(h) * (1.0f / kF8XMainScale)) * kF8XLoScale);
    p.h8 = f32_to_e4m3(x * kF8XHiScale);
    return p;
}

}  // namespace h3d

// TF 1.3 dropout (utils/general.py:139-148) of the lifting stage's FC stacks, and its gradient.  The generator, the counter layout and
// the arithmetic are documented with H3D_DROPOUT_* in include/hand3d_b200.h; tests/dropout_oracle.py restates them in numpy bit for bit,
// so every step is an explicitly rounded fp32 operation.
#include "common.cuh"
#include "philox.cuh"

namespace h3d {

namespace {

template <bool FP16>
__device__ __forceinline__ uint16_t dropout_h16(float v) {
    if (FP16) return __half_as_ushort(__float2half_rn(v));
    return __bfloat16_as_ushort(__float2bfloat16_rn(v));
}
template <bool FP16>
__device__ __forceinline__ float dropout_f32(uint16_t v) {
    if (FP16) return __half2float(__ushort_as_half(v));
    return __uint_as_float((uint32_t)v << 16);
}

// One thread per (row, group of four columns): one Philox block (draw, layer, row, col / 4) gives the four keep bits
// k = floor(keep_prob + u), u = (w >> 40) 2^-24, and y = (x / keep_prob) * k.  PLANES = 0: fp32 y only; 1: bf16, 2: fp16 hi / lo planes
// [rows, stride] as well (lo may be NULL), zero in the columns [cols, stride).  x == y is allowed (in place).
template <int PLANES>
__global__ void dropout_kernel(const float* x, int rows, int cols, float keep_prob, int layer, uint64_t seed, const int64_t* __restrict__ draw,
                               float* y, uint8_t* __restrict__ keep, uint16_t* __restrict__ hi, uint16_t* __restrict__ lo, int stride) {
    const uint64_t d = (uint64_t)*draw;
    const int width = PLANES ? stride : cols;
    const int groups = (width + 3) / 4;
    const int64_t total = (int64_t)rows * groups;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int row = (int)(i / groups), col0 = 4 * (int)(i - (int64_t)row * groups);
        uint64_t c[4] = {d, (uint64_t)layer, (uint64_t)row, (uint64_t)(col0 / 4)};
        if (col0 < cols) philox4x64_10(c, seed, H3D_DROPOUT_STREAM);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int col = col0 + j;
            if (col >= width) break;
            float v = 0.f;
            if (col < cols) {
                const float k = floorf(__fadd_rn(keep_prob, uniform01(c[j])));
                const int64_t e = (int64_t)row * cols + col;
                v = __fmul_rn(__fdiv_rn(x[e], keep_prob), k);
                if (y) y[e] = v;
                if (keep) keep[e] = (uint8_t)k;
            }
            if (PLANES) {
                const int64_t p = (int64_t)row * stride + col;
                const uint16_t h = dropout_h16<PLANES == 2>(v);
                hi[p] = h;
                if (lo) lo[p] = dropout_h16<PLANES == 2>(__fsub_rn(v, dropout_f32<PLANES == 2>(h)));
            }
        }
    }
}

// dx = (dy * k) / keep_prob: TF's Mul gradient, then its RealDiv gradient.
__global__ void dropout_backward_kernel(const float* __restrict__ dy, const uint8_t* __restrict__ keep, int64_t n, float keep_prob,
                                        float* __restrict__ dx) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        dx[i] = __fdiv_rn(__fmul_rn(dy[i], (float)keep[i]), keep_prob);
}

__global__ void dropout_advance_kernel(int64_t* draw) { *draw += 1; }

int grid_for(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div64(n, 256), 132 * 16)); }

}  // namespace

int launch_dropout(const float* x, int rows, int cols, float keep_prob, int layer, uint64_t seed, const int64_t* draw, float* y, uint8_t* keep,
                   Split planes, int stride, Half16 t, cudaStream_t s) {
    if (!planes.hi) {
        dropout_kernel<0><<<grid_for((int64_t)rows * ceil_div(cols, 4)), 256, 0, s>>>(x, rows, cols, keep_prob, layer, seed, draw, y, keep,
                                                                                      nullptr, nullptr, cols);
    } else {
        H3D_REQUIRE(stride >= cols && !planes.l8, "dropout: bad plane arguments");
        const int g = grid_for((int64_t)rows * ceil_div(stride, 4));
        if (t == Half16::FP16) dropout_kernel<2><<<g, 256, 0, s>>>(x, rows, cols, keep_prob, layer, seed, draw, y, keep, planes.hi, planes.lo, stride);
        else dropout_kernel<1><<<g, 256, 0, s>>>(x, rows, cols, keep_prob, layer, seed, draw, y, keep, planes.hi, planes.lo, stride);
    }
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

int launch_dropout_backward(const float* dy, const uint8_t* keep, int64_t n, float keep_prob, float* dx, cudaStream_t s) {
    dropout_backward_kernel<<<grid_for(n), 256, 0, s>>>(dy, keep, n, keep_prob, dx);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

int launch_dropout_advance(int64_t* draw, cudaStream_t s) {
    dropout_advance_kernel<<<1, 1, 0, s>>>(draw);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

}  // namespace h3d

// fp32 CUDA-core kernels: generic NHWC direct convolution (tf.nn.conv2d 'SAME' + bias + leaky ReLU,
// utils/general.py:36-59) used for the layers tensor cores cannot help (Cin = 3 first layers, K = 27;
// Cout = 2 / 21 score-map heads; the tiny stride-2 lifting pyramids), the fully connected layers
// (utils/general.py:113-136) and as the fp32 yard-stick path (H3D_PREC_FP32_FFMA).
#include <cstdlib>

#include "common.cuh"
#include "split_fmt.cuh"

namespace h3d {

namespace {

constexpr int TM = 64;   // output pixels per CTA
constexpr int TN = 64;   // output channels per CTA
constexpr int KC = 16;   // reduction chunk

template <bool FP16>
__device__ __forceinline__ uint16_t to_h16(float v) {
    if (FP16) return __half_as_ushort(__float2half_rn(v));
    return __bfloat16_as_ushort(__float2bfloat16_rn(v));
}
template <bool FP16>
__device__ __forceinline__ float from_h16(uint16_t v) {
    if (FP16) return __half2float(__ushort_as_half(v));
    return __uint_as_float((uint32_t)v << 16);
}

struct ConvGeom {
    int B, H, W, Ho, Wo, Cin, Cout, k, stride, pad_t, pad_l;
    int Cin_total, cin_off, Cout_total, cout_off, Cs_total, cs_off;
    int leaky;
    uint8_t* yl8; uint8_t* yh8;   // fp16_f8c planes (see split_fmt.cuh); yhi then holds fp16
    int k_per_split;     // reduction range handled by one blockIdx.z (multiple of KC); == Ktot when not split
    float* partial;      // split-K: raw partial sums [gridDim.z][M][Cout]
    const int* count;    // counted batch: only images [0, *count) (DirectConvArgs::count); never with split-K
    const int* slots;    // image b of the launch is image slots[b] of x (DirectConvArgs::slots)
};

// VEC: Cin % 16 == 0 and 16-byte aligned input channels -> one tap per K chunk, float4 gathers.
template <bool VEC, bool FP16>
__global__ void __launch_bounds__(256)
conv_direct_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                   float* __restrict__ y, uint16_t* __restrict__ yhi, uint16_t* __restrict__ ylo, ConvGeom g) {
    __shared__ __align__(16) float As[KC][TM + 4];
    __shared__ __align__(16) float Bs[KC][TN + 4];
    const int t = threadIdx.x;
    const int tx = t & 15, ty = t >> 4;
    const int64_t M = (int64_t)(g.count ? min(*g.count, g.B) : g.B) * g.Ho * g.Wo;
    const int64_t m0 = (int64_t)blockIdx.x * TM;
    if (m0 >= M) return;   // counted batch: the whole CTA lies past the last image
    const int n0 = blockIdx.y * TN;
    const int Ktot = g.k * g.k * g.Cin;

    // the pixel this thread gathers for (fixed across the K loop)
    const int a_pix = VEC ? (t >> 2) : (t & 63);
    const int64_t am = m0 + a_pix;
    const bool a_valid = am < M;
    int ab = 0, aoy = 0, aox = 0;
    if (a_valid) {
        aox = (int)(am % g.Wo);
        aoy = (int)((am / g.Wo) % g.Ho);
        ab = (int)(am / ((int64_t)g.Wo * g.Ho));
    }
    const int iy0 = aoy * g.stride - g.pad_t, ix0 = aox * g.stride - g.pad_l;
    const float* xb = x + (int64_t)(g.slots && a_valid ? g.slots[ab] : ab) * g.H * g.W * g.Cin_total + g.cin_off;

    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    const int kk_begin = blockIdx.z * g.k_per_split, kk_end = min(Ktot, kk_begin + g.k_per_split);
    for (int kk0 = kk_begin; kk0 < kk_end; kk0 += KC) {
        // ---- gather A chunk
        if (VEC) {
            const int tap = kk0 / g.Cin, c0 = kk0 - tap * g.Cin;
            const int kh = tap / g.k, kw = tap - kh * g.k;
            const int iy = iy0 + kh, ix = ix0 + kw;
            const int cs = (t & 3) * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (a_valid && iy >= 0 && iy < g.H && ix >= 0 && ix < g.W)
                v = __ldg(reinterpret_cast<const float4*>(xb + ((int64_t)iy * g.W + ix) * g.Cin_total + c0 + cs));
            As[cs + 0][a_pix] = v.x; As[cs + 1][a_pix] = v.y; As[cs + 2][a_pix] = v.z; As[cs + 3][a_pix] = v.w;
        } else {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int ks = (t >> 6) + q * 4;
                const int kk = kk0 + ks;
                float v = 0.f;
                if (a_valid && kk < Ktot) {
                    const int tap = kk / g.Cin, ci = kk - tap * g.Cin;
                    const int kh = tap / g.k, kw = tap - kh * g.k;
                    const int iy = iy0 + kh, ix = ix0 + kw;
                    if (iy >= 0 && iy < g.H && ix >= 0 && ix < g.W) v = __ldg(xb + ((int64_t)iy * g.W + ix) * g.Cin_total + ci);
                }
                As[ks][a_pix] = v;
            }
        }
        // ---- load B chunk (HWIO: row kk, Cout contiguous)
        {
            const int r = t >> 4, c4 = (t & 15) * 4;
            const int kk = kk0 + r;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (kk < Ktot) {
                const float* wr = w + (int64_t)kk * g.Cout + n0 + c4;
                if ((g.Cout & 3) == 0 && n0 + c4 + 3 < g.Cout) {
                    v = __ldg(reinterpret_cast<const float4*>(wr));
                } else {
                    if (n0 + c4 + 0 < g.Cout) v.x = __ldg(wr + 0);
                    if (n0 + c4 + 1 < g.Cout) v.y = __ldg(wr + 1);
                    if (n0 + c4 + 2 < g.Cout) v.z = __ldg(wr + 2);
                    if (n0 + c4 + 3 < g.Cout) v.w = __ldg(wr + 3);
                }
            }
            *reinterpret_cast<float4*>(&Bs[r][c4]) = v;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < KC; ++k) {
            const float4 a = *reinterpret_cast<const float4*>(&As[k][tx * 4]);
            const float4 b = *reinterpret_cast<const float4*>(&Bs[k][ty * 4]);
            const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }

    const int nb = n0 + ty * 4;
    if (g.partial) {   // split-K: raw partial sums, reduced (+ bias, activation) by conv_splitk_reduce_kernel
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int64_t m = m0 + tx * 4 + i;
            if (m >= M) continue;
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (nb + j < g.Cout) g.partial[((int64_t)blockIdx.z * M + m) * g.Cout + nb + j] = acc[i][j];
        }
        return;
    }
    // ---- epilogue: bias + leaky ReLU, fp32 and / or split store
    float bvals[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) bvals[j] = (nb + j < g.Cout) ? __ldg(bias + nb + j) : 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int64_t m = m0 + tx * 4 + i;
        if (m >= M) continue;
        float o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float v = acc[i][j] + bvals[j];
            if (g.leaky) v = fmaxf(v, kNegSlope * v);
            o[j] = v;
        }
        if (y) {
            float* dst = y + m * g.Cout_total + g.cout_off + nb;
            if (nb + 3 < g.Cout && ((g.Cout_total | g.cout_off) & 3) == 0) {
                *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
            } else {
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (nb + j < g.Cout) dst[j] = o[j];
            }
        }
        if (yhi) {
            const int64_t off = m * g.Cs_total + g.cs_off + nb;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                if (nb + j < g.Cout) {
                    if (g.yl8) {
                        const F8cPlanes pl = f32_to_f8c(o[j]);
                        yhi[off + j] = pl.h16; g.yl8[off + j] = pl.l8; g.yh8[off + j] = pl.h8;
                    } else {
                        const uint16_t h = to_h16<FP16>(o[j]);
                        yhi[off + j] = h;
                        if (ylo) ylo[off + j] = to_h16<FP16>(o[j] - from_h16<FP16>(h));
                    }
                }
            }
        }
    }
}

__global__ void conv_splitk_reduce_kernel(const float* __restrict__ part, const float* __restrict__ bias, float* __restrict__ y,
                                          int64_t M, int Cout, int ksplit, int Cout_total, int cout_off, int leaky) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= M * Cout) return;
    float v = 0.f;
    for (int z = 0; z < ksplit; ++z) v += part[(int64_t)z * M * Cout + i];   // fixed order: deterministic
    const int n = (int)(i % Cout);
    v += __ldg(bias + n);
    if (leaky) v = fmaxf(v, kNegSlope * v);
    y[(i / Cout) * Cout_total + cout_off + n] = v;
}

// ---------------------------------------------------------------------------------------------
// First layers (HandSegNet/conv1_1, PoseNet2D/conv1_1): 3x3, Cin = 3, Cout = 64, stride 1.  K = 27 is too small
// for the tensor pipe; the layer is bound by its 64-channel output write, so it runs on CUDA cores with
// register tiling: one CTA = 8 x 32 output pixels, one warp = one image row of the tile, one thread =
// 8 pixels x 8 output channels (64 accumulators).  Weights [27][64] and the haloed input tile live in shared
// memory; all shared loads are 128-bit and warp-broadcast (8 lanes share an address), so the inner loop is
// 192 FFMA per 10 LDS.128.  Stores: the 8 lanes of a pixel write 128 (split) / 256 (fp32) contiguous bytes.
// ---------------------------------------------------------------------------------------------
constexpr int C3_TH = 8, C3_TW = 32, C3_LD = 40, C3_TILES_PER_CTA = 4;   // tile rows, tile cols, padded smem row (pixel x=-1 sits at index 3)

template <bool FP16>
__global__ void __launch_bounds__(256, 2)
conv3x3_c3_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias, float* __restrict__ y,
                  uint16_t* __restrict__ yhi, uint16_t* __restrict__ ylo, uint8_t* __restrict__ yl8, uint8_t* __restrict__ yh8, int B, int H,
                  int W, int Cy_total, int cy_off, int Cs_total, int cs_off, int leaky, const int* __restrict__ count,
                  const int* __restrict__ slots) {
    __shared__ __align__(16) float ws[27][64];
    __shared__ __align__(16) float xs[3][C3_TH + 2][C3_LD];
    const int t = threadIdx.x;
    const int tiles_w = (W + C3_TW - 1) / C3_TW, tiles_h = (H + C3_TH - 1) / C3_TH;
    const int num_tiles = tiles_w * tiles_h * (count ? min(*count, B) : B);   // images are the slowest tile index
    for (int i = t; i < 27 * 64; i += 256) (&ws[0][0])[i] = __ldg(w + i);      // weights staged once per CTA
    for (int i = t; i < 3 * (C3_TH + 2) * C3_LD; i += 256) (&xs[0][0][0])[i] = 0.f;   // alignment padding columns stay zero
    for (int tile = blockIdx.x * C3_TILES_PER_CTA; tile < min(num_tiles, (blockIdx.x + 1) * C3_TILES_PER_CTA); ++tile) {
    const int tw = tile % tiles_w, th = (tile / tiles_w) % tiles_h, b = tile / (tiles_w * tiles_h);
    const int x0 = tw * C3_TW, y0 = th * C3_TH;
    __syncthreads();                                                            // previous tile fully consumed (and ws visible)
    const float* xb = x + (int64_t)(slots ? slots[b] : b) * H * W * 3;
    for (int i = t; i < (C3_TH + 2) * (C3_TW + 2) * 3; i += 256) {              // haloed input tile (contiguous (x, c) reads), zero outside the image
        const int r = i / ((C3_TW + 2) * 3), rem = i - r * ((C3_TW + 2) * 3);
        const int c = rem / 3, ci = rem - c * 3;
        const int gy = y0 - 1 + r, gx = x0 - 1 + c;
        float v = 0.f;
        if (gy >= 0 && gy < H && gx >= 0 && gx < W) v = __ldg(xb + ((int64_t)gy * W + gx) * 3 + ci);
        xs[ci][r][c + 3] = v;
    }
    __syncthreads();
    const int warp = t >> 5, lane = t & 31;
    const int cg = lane & 7, pg = lane >> 3;      // 8 output channels [8cg, 8cg+8), 8 pixels [8pg, 8pg+8) of row `warp`
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
#pragma unroll
        for (int ci = 0; ci < 3; ++ci) {
            float in[16];
            const float4* src = reinterpret_cast<const float4*>(&xs[ci][warp + kh][pg * 8]);
#pragma unroll
            for (int q = 0; q < 4; ++q) { const float4 v = src[q]; in[4 * q] = v.x; in[4 * q + 1] = v.y; in[4 * q + 2] = v.z; in[4 * q + 3] = v.w; }
#pragma unroll
            for (int kw = 0; kw < 3; ++kw) {
                const float4 w0 = *reinterpret_cast<const float4*>(&ws[(kh * 3 + kw) * 3 + ci][cg * 8]);
                const float4 w1 = *reinterpret_cast<const float4*>(&ws[(kh * 3 + kw) * 3 + ci][cg * 8 + 4]);
                const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const float a = in[3 + i + kw];      // pixel 8pg + i, tap kw: x = 8pg + i + kw - 1 -> index 8pg + i + kw + 3
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a, wv[j], acc[i][j]);
                }
            }
        }
    }
    float bv[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) bv[j] = __ldg(bias + cg * 8 + j);
    const int gy = y0 + warp;
    if (gy < H) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int gx = x0 + pg * 8 + i;
        if (gx >= W) continue;
        const int64_t pix = ((int64_t)b * H + gy) * W + gx;
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float v = acc[i][j] + bv[j];
            if (leaky) v = fmaxf(v, kNegSlope * v);
            o[j] = v;
        }
        if (y) {
            float4* dst = reinterpret_cast<float4*>(y + pix * Cy_total + cy_off + cg * 8);
            dst[0] = make_float4(o[0], o[1], o[2], o[3]);
            dst[1] = make_float4(o[4], o[5], o[6], o[7]);
        }
        if (yhi && yl8) {            // fp16 + e4m3 planes (fp16_f8c)
            uint16_t h[8]; uint8_t l8[8], h8[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) { const F8cPlanes pl = f32_to_f8c(o[j]); h[j] = pl.h16; l8[j] = pl.l8; h8[j] = pl.h8; }
            const int64_t off = pix * Cs_total + cs_off + cg * 8;
            *reinterpret_cast<uint4*>(yhi + off) = *reinterpret_cast<const uint4*>(h);
            *reinterpret_cast<uint2*>(yl8 + off) = *reinterpret_cast<const uint2*>(l8);
            *reinterpret_cast<uint2*>(yh8 + off) = *reinterpret_cast<const uint2*>(h8);
        } else if (yhi) {
            uint16_t h[8], l[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) { h[j] = to_h16<FP16>(o[j]); l[j] = to_h16<FP16>(o[j] - from_h16<FP16>(h[j])); }
            const int64_t off = pix * Cs_total + cs_off + cg * 8;
            *reinterpret_cast<uint4*>(yhi + off) = *reinterpret_cast<const uint4*>(h);
            if (ylo) *reinterpret_cast<uint4*>(ylo + off) = *reinterpret_cast<const uint4*>(l);
        }
    }
    }   // gy < H
    }   // tile loop
}

}  // namespace

static bool is_c3_case(const DirectConvArgs& a) {
    return a.Cin == 3 && a.Cin_total == 3 && a.cin_off == 0 && a.k == 3 && a.stride == 1 && a.Cout == 64 &&
           (!a.y || ((a.Cout_total % 4) == 0 && (a.cout_off % 4) == 0)) && (!a.ys.hi || ((a.Cs_total % 8) == 0 && (a.cs_off % 8) == 0));
}

// Launch geometry + split-K policy shared by the launcher and by conv_direct_geometry().
static void plan_direct(const DirectConvArgs& a, ConvGeom* gp, dim3* gridp, int* ksplitp) {
    ConvGeom& g = *gp;
    g.B = a.B; g.H = a.H; g.W = a.W; g.Cin = a.Cin; g.Cout = a.Cout; g.k = a.k; g.stride = a.stride;
    g.Ho = ceil_div(a.H, a.stride); g.Wo = ceil_div(a.W, a.stride);
    const int tot_h = std::max((g.Ho - 1) * a.stride + a.k - a.H, 0), tot_w = std::max((g.Wo - 1) * a.stride + a.k - a.W, 0);
    g.pad_t = tot_h / 2; g.pad_l = tot_w / 2;   // TF 'SAME': the odd pixel goes to the bottom / right (SURVEY 9.1)
    g.Cin_total = a.Cin_total; g.cin_off = a.cin_off; g.Cout_total = a.Cout_total; g.cout_off = a.cout_off;
    g.Cs_total = a.Cs_total; g.cs_off = a.cs_off; g.leaky = a.leaky;
    g.yl8 = a.ys.l8; g.yh8 = a.ys.h8;
    g.count = a.count; g.slots = a.slots;
    const int64_t M = (int64_t)g.B * g.Ho * g.Wo;
    dim3 grid((unsigned)ceil_div64(M, TM), (unsigned)ceil_div(a.Cout, TN));
    const int Ktot = a.k * a.k * a.Cin;
    g.k_per_split = (int)align_up(Ktot, KC);
    g.partial = nullptr;
    int ksplit = 1;
    const int ctas = (int)(grid.x * grid.y);
    if (a.splitk_scratch && !a.count && a.y && !a.ys.hi && ctas < 296 && Ktot >= 256) {
        // tiny spatial maps (the stride-2 lifting pyramids): too few tiles to fill 132 SMs -> split the reduction
        ksplit = std::min(ceil_div(Ktot, 128), std::max(1, 592 / ctas));
        if (ksplit > 1 && (int64_t)ksplit * M * a.Cout <= a.splitk_scratch_floats) {
            g.k_per_split = (int)align_up(ceil_div(Ktot, ksplit), KC);
            ksplit = ceil_div(Ktot, g.k_per_split);
            if (ksplit > 1) { g.partial = a.splitk_scratch; grid.z = ksplit; }
        } else {
            ksplit = 1;
        }
    }
    *gridp = grid; *ksplitp = ksplit;
}

// The kernel launch_conv_direct runs (H3D_DIRECT_*).
static int direct_kernel(const DirectConvArgs& a) {
    if (is_c3_case(a))   // split planes only (not fp16_f8c): the tensor-core version
        return !a.y && a.ys.hi && !a.ys.l8 && !tc_tuning().c3_ffma ? H3D_DIRECT_C3_TC : H3D_DIRECT_C3_FFMA;
    const bool vec = (a.Cin % KC == 0) && (a.Cin_total % 4 == 0) && (a.cin_off % 4 == 0) && (((uintptr_t)a.x & 15) == 0);
    return vec ? H3D_DIRECT_VEC : H3D_DIRECT_SCALAR;
}

static int c3_ctas(const DirectConvArgs& a) { return ceil_div(ceil_div(a.W, C3_TW) * ceil_div(a.H, C3_TH) * a.B, C3_TILES_PER_CTA); }

void conv_direct_geometry(const DirectConvArgs& a, int* out) {
    const int kernel = direct_kernel(a);
    out[0] = kernel;
    if (kernel == H3D_DIRECT_C3_TC || kernel == H3D_DIRECT_C3_FFMA) {
        const int ctas = kernel == H3D_DIRECT_C3_FFMA ? c3_ctas(a) : 0;
        out[1] = ctas; out[2] = out[3] = ctas ? 1 : 0; out[4] = 1; out[5] = 27;
        return;
    }
    ConvGeom g; dim3 grid; int ksplit;
    plan_direct(a, &g, &grid, &ksplit);
    out[1] = (int)grid.x; out[2] = (int)grid.y; out[3] = (int)grid.z; out[4] = ksplit; out[5] = g.k_per_split;
}

int launch_conv_direct(const DirectConvArgs& a, cudaStream_t s) {
    H3D_REQUIRE(a.k >= 1 && a.stride >= 1 && a.Cin >= 1 && a.Cout >= 1, "conv_direct: bad geometry");
    const int kernel = direct_kernel(a);
    if (kernel == H3D_DIRECT_C3_TC)
        return launch_conv_c3_tc(a.x, a.w, a.bias, a.ys, a.Cs_total, a.cs_off, a.B, a.H, a.W, a.leaky, a.half, s, a.err_flag, a.count, a.slots);
    if (kernel == H3D_DIRECT_C3_FFMA) {
        const int tiles = c3_ctas(a);
        if (a.half == Half16::FP16)
            conv3x3_c3_kernel<true><<<tiles, 256, 0, s>>>(a.x, a.w, a.bias, a.y, a.ys.hi, a.ys.lo, a.ys.l8, a.ys.h8, a.B, a.H, a.W, a.Cout_total, a.cout_off, a.Cs_total, a.cs_off, a.leaky, a.count, a.slots);
        else
            conv3x3_c3_kernel<false><<<tiles, 256, 0, s>>>(a.x, a.w, a.bias, a.y, a.ys.hi, a.ys.lo, a.ys.l8, a.ys.h8, a.B, a.H, a.W, a.Cout_total, a.cout_off, a.Cs_total, a.cs_off, a.leaky, a.count, a.slots);
        H3D_CHECK_LAUNCH();
        return H3D_OK;
    }
    ConvGeom g; dim3 grid; int ksplit;
    plan_direct(a, &g, &grid, &ksplit);
    const int64_t M = (int64_t)g.B * g.Ho * g.Wo;
    const bool vec = kernel == H3D_DIRECT_VEC;
    const bool fp16 = a.half == Half16::FP16;
#define LAUNCH(V, F) conv_direct_kernel<V, F><<<grid, 256, 0, s>>>(a.x, a.w, a.bias, a.y, a.ys.hi, a.ys.lo, g)
    if (vec) { if (fp16) LAUNCH(true, true); else LAUNCH(true, false); }
    else     { if (fp16) LAUNCH(false, true); else LAUNCH(false, false); }
#undef LAUNCH
    H3D_CHECK_LAUNCH();
    if (ksplit > 1) {
        conv_splitk_reduce_kernel<<<(unsigned)ceil_div64(M * a.Cout, 256), 256, 0, s>>>(a.splitk_scratch, a.bias, a.y, M, a.Cout, ksplit,
                                                                                 a.Cout_total, a.cout_off, a.leaky);
        H3D_CHECK_LAUNCH();
    }
    return H3D_OK;
}

// ---------------------------------------------------------------------------------------------
// NetworkOps.fully_connected(_relu): y = x @ W[in,out] + b (+ leaky).  M = batch is tiny, so the op is a
// weight-streaming problem: split-K over many CTAs (32 batch rows x 64 outputs x one K slice each, W read
// with coalesced 256-byte rows exactly once per batch tile), partial sums to a scratch buffer, then a
// fixed-order reduction + bias + leaky ReLU (deterministic: no floating-point atomics).
// ---------------------------------------------------------------------------------------------
constexpr int FCB = 32, FCN = 64, FCK = 32;

__global__ void __launch_bounds__(256)
fc_splitk_kernel(const float* __restrict__ x, const float* __restrict__ w, float* __restrict__ part, int B, int in_f, int out_f,
                 int x_stride, int k_per_split) {
    __shared__ float xs[FCB][FCK + 1];
    const int t = threadIdx.x;
    const int n = blockIdx.x * FCN + (t & 63);
    const int rb = (t >> 6) * 8;            // 8 batch rows per thread
    const int b0 = blockIdx.z * FCB;
    const int ks = blockIdx.y;
    const int kbeg = ks * k_per_split, kend = min(in_f, kbeg + k_per_split);
    float acc[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) acc[r] = 0.f;
    for (int k0 = kbeg; k0 < kend; k0 += FCK) {
        for (int i = t; i < FCB * FCK; i += 256) {
            const int r = i / FCK, c = i - r * FCK;
            xs[r][c] = (b0 + r < B && k0 + c < kend) ? __ldg(x + (int64_t)(b0 + r) * x_stride + k0 + c) : 0.f;
        }
        __syncthreads();
        if (n < out_f) {
            const int kmax = min(FCK, kend - k0);
#pragma unroll 8
            for (int k = 0; k < kmax; ++k) {
                const float wv = __ldg(w + (int64_t)(k0 + k) * out_f + n);
#pragma unroll
                for (int r = 0; r < 8; ++r) acc[r] = fmaf(xs[rb + r][k], wv, acc[r]);
            }
        }
        __syncthreads();
    }
    if (n < out_f) {
#pragma unroll
        for (int r = 0; r < 8; ++r) {
            const int b = b0 + rb + r;
            if (b < B) part[((int64_t)ks * B + b) * out_f + n] = acc[r];
        }
    }
}

__global__ void fc_reduce_kernel(const float* __restrict__ part, const float* __restrict__ bias, float* __restrict__ y, int B,
                                 int out_f, int ksplit, int leaky) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * out_f) return;
    float v = 0.f;
    for (int ks = 0; ks < ksplit; ++ks) v += part[(int64_t)ks * B * out_f + i];   // fixed order
    v += __ldg(bias + (i % out_f));
    if (leaky) v = fmaxf(v, kNegSlope * v);
    y[i] = v;
}

int fc_ksplit(int B, int in_f, int out_f) {
    const int ctas = ceil_div(out_f, FCN) * ceil_div(B, FCB);
    int ks = std::max(1, std::min(ceil_div(in_f, 64), 296 / std::max(1, ctas)));
    return ks;
}
int64_t fc_scratch_floats(int B, int in_f, int out_f) { return (int64_t)fc_ksplit(B, in_f, out_f) * B * out_f; }
static int fc_k_per_split(int in_f, int ksplit) { return (int)align_up(ceil_div(in_f, ksplit), FCK); }
void fc_geometry(int B, int in_f, int out_f, int* out) {
    const int ksplit = fc_ksplit(B, in_f, out_f);
    out[0] = ksplit; out[1] = fc_k_per_split(in_f, ksplit); out[2] = ceil_div(out_f, FCN); out[3] = ksplit; out[4] = ceil_div(B, FCB);
}

int launch_fc(const float* x, const float* w, const float* bias, float* y, float* scratch, int64_t scratch_floats, int B, int in_f,
              int out_f, int leaky, int x_stride, cudaStream_t s) {
    const int ksplit = fc_ksplit(B, in_f, out_f);
    H3D_REQUIRE((int64_t)ksplit * B * out_f <= scratch_floats, "fully_connected %d -> %d at B=%d: split-K needs %lld scratch floats, have %lld",
                in_f, out_f, B, (long long)ksplit * B * out_f, (long long)scratch_floats);
    const int k_per_split = fc_k_per_split(in_f, ksplit);
    dim3 grid(ceil_div(out_f, FCN), ksplit, ceil_div(B, FCB));
    fc_splitk_kernel<<<grid, 256, 0, s>>>(x, w, scratch, B, in_f, out_f, x_stride, k_per_split);
    H3D_CHECK_LAUNCH();
    fc_reduce_kernel<<<ceil_div(B * out_f, 256), 256, 0, s>>>(scratch, bias, y, B, out_f, ksplit, leaky);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

// tf.reshape([B,-1]) of the NHWC feature map + tf.concat([x, hand_side], 1)  (nets/...:262-263,297-298)
__global__ void concat_handside_kernel(const float* __restrict__ feat, const float* __restrict__ hs, float* __restrict__ out,
                                       int B, int n) {
    const int64_t total = (int64_t)B * (n + 2);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % (n + 2));
        const int b = (int)(i / (n + 2));
        out[i] = c < n ? feat[(int64_t)b * n + c] : hs[2 * b + (c - n)];
    }
}
// same, emitting the 16-bit split planes [B, Kpad] (zero padded) that feed the tensor-core FC stack
template <bool FP16>
__global__ void concat_handside_split_kernel(const float* __restrict__ feat, const float* __restrict__ hs, uint16_t* __restrict__ hi,
                                             uint16_t* __restrict__ lo, int B, int n, int Kpad) {
    const int64_t total = (int64_t)B * Kpad;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % Kpad);
        const int b = (int)(i / Kpad);
        const float v = c < n ? feat[(int64_t)b * n + c] : (c < n + 2 ? hs[2 * b + (c - n)] : 0.f);
        const uint16_t h = to_h16<FP16>(v);
        hi[i] = h;
        if (lo) lo[i] = to_h16<FP16>(v - from_h16<FP16>(h));
    }
}
int launch_concat_handside_split(const float* feat, const float* hand_side, Split out, int B, int feat_n, int Kpad, Half16 t, cudaStream_t s) {
    H3D_REQUIRE(out.hi && !out.l8 && Kpad >= feat_n + 2, "concat_handside_split: bad argument");
    const int blocks = (int)std::min<int64_t>(ceil_div64((int64_t)B * Kpad, 256), 1024);
    if (t == Half16::FP16) concat_handside_split_kernel<true><<<blocks, 256, 0, s>>>(feat, hand_side, out.hi, out.lo, B, feat_n, Kpad);
    else concat_handside_split_kernel<false><<<blocks, 256, 0, s>>>(feat, hand_side, out.hi, out.lo, B, feat_n, Kpad);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}
int launch_concat_handside(const float* feat, const float* hand_side, float* out, int B, int feat_n, cudaStream_t s) {
    const int64_t total = (int64_t)B * (feat_n + 2);
    concat_handside_kernel<<<(int)std::min<int64_t>(ceil_div64(total, 256), 1024), 256, 0, s>>>(feat, hand_side, out, B, feat_n);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

}  // namespace h3d

// Hopper (sm_90a) implicit-GEMM convolution on the tensor cores (tf.nn.conv2d 'SAME' stride 1 + bias + leaky ReLU,
// utils/general.py:36-59), im2col-free:
//
//   D[M = 128 output pixels, N = BN output channels] += A[M, K] * B[N, K]^T,   K = kh*kw*Cin
//
// * A is never materialised.  For filter tap (kh, kw) and 64-channel chunk c the A tile is the 4-D TMA
//   box {64 ch, TW, TH, TB} of the NHWC activation tensor at (c, w0+kw-pad, h0+kh-pad, b0): TMA's
//   out-of-bounds zero fill (negative / past-the-end coordinates) implements the 'SAME' zero padding
//   and never leaks pixels across images.  The box lands in shared memory as 128 rows x 128 bytes with
//   the 128-byte swizzle, which is exactly the K-major SWIZZLE_128B layout wgmma reads.
// * B tiles are 2-D TMA boxes {64, BN} of the pre-packed K-major weights [Cout][kh][kw][Cin].
// * fp32 parity on 16-bit tensor cores: activations and weights are stored as two 16-bit planes
//   x = hi + lo; each K block issues hi*hi + hi*lo + lo*hi (3 passes) into the same fp32 register
//   accumulator.  Per operand the split keeps 16 (bf16) or 22 (fp16) significant bits, so the dropped lo*lo term is ~2^-16
//   (bf16) or ~2^-22 (fp16) of a product -- as long as lo stays a normal number.  bf16 has fp32's exponent range; fp16's
//   ends at 2^-14, so fp16 weight planes are packed with a per-output-channel power-of-two shift that the epilogue un-does
//   (split_fmt.cuh), and fp16 activations keep the full split only for |x| >= ~2^-3 (below, lo is subnormal and the error
//   grows towards single-pass fp16's; DESIGN.md section 6.1 gives the measured ranges).  PASSES == 1 is the plain 16-bit
//   path; PASSES == 4 is one fp16 pass plus two e4m3 correction passes (split_fmt.cuh).
// * Warp-specialised persistent CTAs of three warpgroups: warpgroup 0 is the TMA producer (one elected lane of
//   its first warp issues), warpgroups 1 and 2 each own 64 rows of the 128-pixel tile and issue wgmma.mma_async
//   on them.  A ring of shared-memory stages with full / empty mbarriers decouples the two sides.
// * The tensor core adds into its fp32 accumulator with truncation, an error that grows with the number of
//   accumulation steps; K is therefore cut into chunks of chunk_kb blocks whose partial sums are folded into a second
//   set of fp32 registers with round-to-nearest adds.
// * Epilogue: the fp32 tile goes through a shared-memory staging buffer so that each thread then owns one pixel row
//   and 32 consecutive channels (bias, leaky ReLU, fused 2x2 max-pool or stride-2 sub-sampling, split-plane or fp32
//   stores: epilogue_store32).
#include <cuda.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "split_fmt.cuh"
#include "wgmma_common.cuh"

namespace h3d {

namespace {

constexpr int BM = 128;           // pixels per tile (two warpgroups x wgmma M = 64)
constexpr int BK = 64;            // K elements per stage (= 128 bytes = one swizzle span)
constexpr int kThreads = 384;     // warpgroup 0: TMA producer, warpgroups 1-2: wgmma + epilogue
constexpr int kConsumerThreads = 256;
constexpr int A_TILE_BYTES = BM * BK * 2;
constexpr int STG_COLS = 64;                               // channels per round through the epilogue staging buffer
constexpr int STG_PITCH = STG_COLS + 1;                    // floats per staged row (odd: conflict-free row-wise reads)
constexpr int STG_BYTES = BM * STG_PITCH * 4;
constexpr int kSmemBudget = 227 * 1024 - 2048 - STG_BYTES; // ring stages; 2 KB: alignment slack + barriers

// PASSES: 1 = one 16-bit pass; 3 = hi/lo 16-bit planes, three passes; 4 = fp16 plane + two e4m3 planes (each half the bytes),
// one fp16 pass + two fp8 passes.  Modes 3 and 4 stage the same number of bytes.
__host__ __device__ constexpr int stage_bytes(int BN, int PASSES) { return (PASSES >= 3 ? 2 : 1) * (A_TILE_BYTES + BN * BK * 2); }
__host__ __device__ constexpr int num_stages(int BN, int PASSES) {
    return kSmemBudget / stage_bytes(BN, PASSES) > 8 ? 8 : kSmemBudget / stage_bytes(BN, PASSES);
}
__host__ __device__ constexpr int smem_bytes(int BN, int PASSES) { return num_stages(BN, PASSES) * stage_bytes(BN, PASSES) + STG_BYTES + 2048; }

struct TcParams {
    const float* bias;
    uint16_t* y_hi; uint16_t* y_lo; uint8_t* y_l8; uint8_t* y_h8; int Cy_total, cy_off;
    float corr_scale;   // mode 4: 2^-(10+b), un-does the pre-scaling of the operand planes
    float* yf; int Cyf_total, cyf_off;
    int B, H, W, k, pad, cin_chunks;
    int TW, TH, TB, tiles_w, tiles_h, n_tiles, num_tiles;
    int n_valid;    // number of real output channels (Cout); channels [n_valid, Cout_pad) are padding and never stored
    int pool;       // 1: fuse NetworkOps.max_pool (2x2 / 2) into the epilogue; 2: stride-2 'SAME' convolution (store the odd pixels
                    // of the stride-1 result); outputs are [B, H/2, W/2, C] in both modes
    int chunk_kb;   // K blocks accumulated inside the tensor core before the partial sum is folded into the fp32 registers
    int leaky;
    int* err_flag;
    const float* w_scale;   // fp16 weight planes (PASSES 1 / 3): [Cout_pad] 2^-s per output channel (split_fmt.cuh)
    const int* count;       // NULL, or a device int: only images [0, *count) are computed (read after the grid-dependency wait)
};

// The tile-loop bound and the image bound of a (possibly counted) launch.  The image-group index varies slowest in the tile index, so
// the tiles of the first n images are the prefix [0, ceil(n / TB) * tiles_w * tiles_h * n_tiles) of [0, num_tiles).
__device__ __forceinline__ int counted_images(const TcParams& p) { return p.count ? min(*p.count, p.B) : p.B; }
__device__ __forceinline__ int counted_tiles(const TcParams& p, int nb) {
    return p.count ? min(p.num_tiles, (nb + p.TB - 1) / p.TB * p.tiles_w * p.tiles_h * p.n_tiles) : p.num_tiles;
}

// bias + leaky ReLU + store of 32 consecutive output channels [n, n+32) of one pixel (fp32 and / or hi-lo split planes).
// w_scale (fp16 weight planes): [n, n+32) per-channel factors 2^-s that un-do the weight shift, in global memory (read through the
// read-only path, as the bias) or, with SMEM_SCALE, in shared memory.
// With p.pool the 2x2 max-pool partners of a pixel are lanes (lane ^ 1) and (lane ^ TW) of the same warp (tile rows are
// ordered w-fastest and TW <= 16), so pooling is two warp shuffles per value; the lane with even (w, h) stores.
template <int PASSES, bool FP16, bool SMEM_SCALE = false>
__device__ __forceinline__ void epilogue_store32(const TcParams& p, const float* a, int64_t pix, int n, bool valid, const float* w_scale) {
    float f[32];
    const float4* bp = reinterpret_cast<const float4*>(p.bias + n);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        const float4 bv = __ldg(bp + q);
        if (PASSES == 4) {   // un-do the operand pre-scaling (exact power of two)
            f[4 * q + 0] = fmaf(a[4 * q + 0], p.corr_scale, bv.x);
            f[4 * q + 1] = fmaf(a[4 * q + 1], p.corr_scale, bv.y);
            f[4 * q + 2] = fmaf(a[4 * q + 2], p.corr_scale, bv.z);
            f[4 * q + 3] = fmaf(a[4 * q + 3], p.corr_scale, bv.w);
        } else if (FP16) {   // un-do the per-channel weight shift (exact power of two)
            const float4 sv = SMEM_SCALE ? reinterpret_cast<const float4*>(w_scale + n)[q] : __ldg(reinterpret_cast<const float4*>(w_scale + n) + q);
            f[4 * q + 0] = fmaf(a[4 * q + 0], sv.x, bv.x);
            f[4 * q + 1] = fmaf(a[4 * q + 1], sv.y, bv.y);
            f[4 * q + 2] = fmaf(a[4 * q + 2], sv.z, bv.z);
            f[4 * q + 3] = fmaf(a[4 * q + 3], sv.w, bv.w);
        } else {
            f[4 * q + 0] = a[4 * q + 0] + bv.x;
            f[4 * q + 1] = a[4 * q + 1] + bv.y;
            f[4 * q + 2] = a[4 * q + 2] + bv.z;
            f[4 * q + 3] = a[4 * q + 3] + bv.w;
        }
    }
    if (p.leaky) {
#pragma unroll
        for (int q = 0; q < 32; ++q) f[q] = fmaxf(f[q], kNegSlope * f[q]);
    }
    if (p.pool == 1) {
#pragma unroll
        for (int q = 0; q < 32; ++q) {
            f[q] = fmaxf(f[q], __shfl_xor_sync(0xFFFFFFFFu, f[q], 1));
            f[q] = fmaxf(f[q], __shfl_xor_sync(0xFFFFFFFFu, f[q], p.TW));
        }
    }
    if (!valid) return;
    if (n + 32 > p.n_valid) {   // Cout not a multiple of 32 (score-map heads 2 / 21, lifting 32-channel layers): masked scalar fp32 tail
        const int cnt = p.n_valid - n;   // <= 0: this 32-channel group is padding only
        if (p.yf && cnt > 0) {
            float* dst = p.yf + pix * p.Cyf_total + p.cyf_off + n;
#pragma unroll
            for (int q = 0; q < 32; ++q)
                if (q < cnt) dst[q] = f[q];
        }
        // the split planes carry Cout_pad channels: padding channels are written as exact zeros (they are the next layer's K padding)
#pragma unroll
        for (int q = 0; q < 32; ++q)
            if (q >= cnt) f[q] = 0.f;
    } else if (p.yf) {
        if (((p.Cyf_total | p.cyf_off) & 3) == 0) {
            float4* dst = reinterpret_cast<float4*>(p.yf + pix * p.Cyf_total + p.cyf_off + n);
#pragma unroll
            for (int q = 0; q < 8; ++q) dst[q] = make_float4(f[4 * q], f[4 * q + 1], f[4 * q + 2], f[4 * q + 3]);
        } else {   // row stride not a multiple of 16 bytes (e.g. the 63-wide fc_xyz output): scalar stores
            float* dst = p.yf + pix * p.Cyf_total + p.cyf_off + n;
#pragma unroll
            for (int q = 0; q < 32; ++q) dst[q] = f[q];
        }
    }
    if (p.y_hi) {
        const int64_t off = pix * p.Cy_total + p.cy_off + n;
        uint4* dh = reinterpret_cast<uint4*>(p.y_hi + off);
        uint4* dl = reinterpret_cast<uint4*>(p.y_lo + off);
#pragma unroll
        for (int g = 0; g < 4; ++g) {
            uint32_t hi[4], lo[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                float x0 = f[8 * g + 2 * q], x1 = f[8 * g + 2 * q + 1];
                if (PASSES == 4) {   // main plane pre-scaled by 2^5, saturating (must match f32_to_f8c)
                    x0 = fminf(fmaxf(x0 * kF8XMainScale, -65504.f), 65504.f);
                    x1 = fminf(fmaxf(x1 * kF8XMainScale, -65504.f), 65504.f);
                }
                hi[q] = pack_hi2<FP16>(x0, x1);
                if (PASSES == 3) {
                    const float2 r = unpack2<FP16>(hi[q]);
                    lo[q] = pack_hi2<FP16>(x0 - r.x, x1 - r.y);
                }
            }
            dh[g] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
            if (PASSES == 3 && p.y_lo) dl[g] = make_uint4(lo[0], lo[1], lo[2], lo[3]);
        }
        if (PASSES == 4) {   // e4m3 residual and coarse planes: 32 bytes each
            uint32_t l8[8], h8[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                uint32_t wl = 0, wh = 0;
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const F8cPlanes pl = f32_to_f8c(f[4 * q + e]);
                    wl |= (uint32_t)pl.l8 << (8 * e); wh |= (uint32_t)pl.h8 << (8 * e);
                }
                l8[q] = wl; h8[q] = wh;
            }
            uint4* d8l = reinterpret_cast<uint4*>(p.y_l8 + off);
            uint4* d8h = reinterpret_cast<uint4*>(p.y_h8 + off);
            d8l[0] = make_uint4(l8[0], l8[1], l8[2], l8[3]); d8l[1] = make_uint4(l8[4], l8[5], l8[6], l8[7]);
            d8h[0] = make_uint4(h8[0], h8[1], h8[2], h8[3]); d8h[1] = make_uint4(h8[4], h8[5], h8[6], h8[7]);
        }
    }
}

// ------------------------------------------------------------------------------------------ main loop
// Shared-memory ring of the warp-specialised kernels.  Stage layout:
//   PASSES 1: [A_hi | B_hi];  PASSES 3: [A_hi | A_lo | B_hi | B_lo];
//   PASSES 4: [A fp16 16K | A l8 8K | A h8 8K | B fp16 | B h8 | B l8]  (e4m3 tiles have 64-byte rows)
template <int BN, int PASSES>
struct RingCfg {
    static constexpr int STAGES = num_stages(BN, PASSES);
    static constexpr int STAGE_BYTES = stage_bytes(BN, PASSES);
    static constexpr int B_TILE_BYTES = BN * BK * 2;
    static constexpr int A8_TILE_BYTES = BM * BK, B8_TILE_BYTES = BN * BK;
    static_assert(STAGES >= 3, "the consumers hold two stages while the producer refills a third");
};

// One K block: A box at (a0, a1, a2, a3) of the 4-D activation maps, B box at (kcol, n0) of the weight maps.
// Mode 4 map slots: x_lo = x residual (e4m3), x_h8 = x coarse (e4m3), w_lo = w coarse (e4m3), w_l8 = w residual (e4m3).
template <int BN, int PASSES>
__device__ __forceinline__ void produce_kblock(Ring& r, const CUtensorMap* x_hi, const CUtensorMap* x_lo, const CUtensorMap* x_h8,
                                               const CUtensorMap* w_hi, const CUtensorMap* w_lo, const CUtensorMap* w_l8,
                                               int a0, int a1, int a2, int a3, int kcol, int n0, int* err_flag) {
    using C = RingCfg<BN, PASSES>;
    mbar_wait(&r.empty[r.stage], r.phase ^ 1, err_flag, 1);
    H3D_SKEW(SKEW_PRODUCER, r.stage + r.phase * C::STAGES);
    if (elect_one()) {
        uint8_t* st = r.base + r.stage * C::STAGE_BYTES;
        uint64_t* fb = &r.full[r.stage];
        mbar_expect_tx(fb, C::STAGE_BYTES);
        tma_load_4d(x_hi, st, fb, a0, a1, a2, a3);
        tma_load_2d(w_hi, st + (PASSES >= 3 ? 2 : 1) * A_TILE_BYTES, fb, kcol, n0);
        if (PASSES == 3) {
            tma_load_4d(x_lo, st + A_TILE_BYTES, fb, a0, a1, a2, a3);
            tma_load_2d(w_lo, st + 2 * A_TILE_BYTES + C::B_TILE_BYTES, fb, kcol, n0);
        }
        if (PASSES == 4) {
            tma_load_4d(x_lo, st + A_TILE_BYTES, fb, a0, a1, a2, a3);
            tma_load_4d(x_h8, st + A_TILE_BYTES + C::A8_TILE_BYTES, fb, a0, a1, a2, a3);
            tma_load_2d(w_lo, st + 2 * A_TILE_BYTES + C::B_TILE_BYTES, fb, kcol, n0);
            tma_load_2d(w_l8, st + 2 * A_TILE_BYTES + C::B_TILE_BYTES + C::B8_TILE_BYTES, fb, kcol, n0);
        }
    }
    __syncwarp();
    if (++r.stage == C::STAGES) { r.stage = 0; r.phase ^= 1; }
}

// All K blocks of one tile for the 64 rows of warpgroup wg (0 / 1): racc[BN / 2] = the fp32 accumulator fragment of wgmma
// (n8 block j: racc[4j], racc[4j+1] = row 16 warp + lane / 4, columns 8j + 2 (lane % 4) + {0, 1}; racc[4j+2..3] = row + 8).
// Every chunk of chunk_kb K blocks starts a fresh tensor-core accumulation and is added into racc with round-to-nearest.
// The e4m3 passes of mode 4 accumulate into registers of their own: an fp8 wgmma keeps fewer accumulator bits than an fp16 one,
// and adding them to the fp16 pass's accumulator would round that sum to the shorter format on every instruction.
// A stage is released once the wgmma group that read it has completed: one group stays in flight while the next one is issued.
template <int BN, int PASSES, bool FP16>
__device__ __forceinline__ void mma_tile(Ring& r, int kblocks, int chunk_kb, float* racc, int wg, int lane, int* err_flag) {
    using C = RingCfg<BN, PASSES>;
    constexpr int NR = BN / 2;
    constexpr int NR8 = PASSES == 4 ? NR : 1;
    float acc[NR], acc8[NR8];
#pragma unroll
    for (int i = 0; i < NR; ++i) acc[i] = 0.f;
#pragma unroll
    for (int i = 0; i < NR8; ++i) acc8[i] = 0.f;
    for (int kb0 = 0; kb0 < kblocks; kb0 += chunk_kb) {
        const int kb1 = min(kblocks, kb0 + chunk_kb);
        int pend = -1;
        for (int kb = kb0; kb < kb1; ++kb) {
            mbar_wait(&r.full[r.stage], r.phase, err_flag, 3);
            H3D_SKEW(SKEW_CONSUMER, kb);
            const uint32_t sa = smem_u32(r.base + r.stage * C::STAGE_BYTES);
            const uint32_t a_rows = (uint32_t)wg * 64 * 128;   // this warpgroup's 64 rows of the A tile
            const uint64_t a_hi = desc_sw128(sa + a_rows);
            const uint64_t a_lo = desc_sw128(sa + A_TILE_BYTES + a_rows);
            const uint64_t b_hi = desc_sw128(sa + (PASSES >= 3 ? 2 : 1) * A_TILE_BYTES);
            const uint64_t b_lo = desc_sw128(sa + 2 * A_TILE_BYTES + C::B_TILE_BYTES);
            fence_regs<NR>(acc);
            fence_regs<NR8>(acc8);
            wgmma_fence();
#pragma unroll
            for (int j = 0; j < BK / 16; ++j) {
                const uint64_t koff = (uint64_t)j * 2;   // + 32 bytes per K step of 16 (descriptor addresses are in 16-byte units)
                mma16<BN, FP16>(acc, a_hi + koff, b_hi + koff, (uint32_t)((kb > kb0) | (j != 0)));
                if (PASSES == 3) {
                    mma16<BN, FP16>(acc, a_hi + koff, b_lo + koff, 1u);
                    mma16<BN, FP16>(acc, a_lo + koff, b_hi + koff, 1u);
                }
            }
            if (PASSES == 4) {   // two e4m3 correction passes (K = 32 per instruction: 32 bytes per row), same accumulator
                const uint32_t a8_rows = (uint32_t)wg * 64 * 64;
                const uint64_t a_l8 = desc_sw64(sa + A_TILE_BYTES + a8_rows);
                const uint64_t a_h8 = desc_sw64(sa + A_TILE_BYTES + C::A8_TILE_BYTES + a8_rows);
                const uint64_t b_h8 = desc_sw64(sa + 2 * A_TILE_BYTES + C::B_TILE_BYTES);
                const uint64_t b_l8 = desc_sw64(sa + 2 * A_TILE_BYTES + C::B_TILE_BYTES + C::B8_TILE_BYTES);
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const uint64_t koff = (uint64_t)j * 2;
                    mma8<BN>(acc8, a_l8 + koff, b_h8 + koff, (uint32_t)((kb > kb0) | (j != 0)));
                    mma8<BN>(acc8, a_h8 + koff, b_l8 + koff, 1u);
                }
            }
            wgmma_commit();
            fence_regs<NR>(acc);
            fence_regs<NR8>(acc8);
            H3D_SKEW(SKEW_COMMIT, kb);
            wgmma_wait<1>();
            if (pend >= 0 && lane == 0) mbar_arrive(&r.empty[pend]);
            pend = r.stage;
            if (++r.stage == C::STAGES) { r.stage = 0; r.phase ^= 1; }
        }
        wgmma_wait<0>();
        if (lane == 0) mbar_arrive(&r.empty[pend]);
        fence_regs<NR>(acc);
        fence_regs<NR8>(acc8);
        if constexpr (PASSES == 4) {
#pragma unroll
            for (int i = 0; i < NR; ++i) acc[i] += acc8[i];
        }
        if (kb0 == 0) {
#pragma unroll
            for (int i = 0; i < NR; ++i) racc[i] = acc[i];
        } else {
#pragma unroll
            for (int i = 0; i < NR; ++i) racc[i] += acc[i];
        }
    }
}

// Epilogue of one tile: the two warpgroups' fragments go through the staging buffer (64 channels per round); consumer thread ct
// (0..255) then owns tile row ct % 128 and channels [32 (ct / 128), +32) of the round, so the 2x2 pooling partners of a pixel are
// lanes of one warp as epilogue_store32 requires.  pix_of(row, &pix, &valid) maps a tile row to its output pixel.
template <int BN, int PASSES, bool FP16, class PixOf, bool SMEM_SCALE = false>
__device__ __forceinline__ void store_tile(const TcParams& p, const float* racc, float* stg, int ct, int n0, PixOf pix_of,
                                           const float* w_scale) {
    const int wg = ct >> 7, tt = ct & 127;
    const int r0 = wg * 64 + (tt >> 5) * 16 + ((tt & 31) >> 2);
    const int cq = 2 * (tt & 3);
    const int row = ct & 127, half = ct >> 7;
    int64_t pix; bool valid;
    pix_of(row, pix, valid);
#pragma unroll
    for (int rnd = 0; rnd < BN / STG_COLS; ++rnd) {
        H3D_SKEW(SKEW_EPILOGUE, 2 * rnd);
        named_bar_sync(1, kConsumerThreads);   // the previous round's readers are done with the buffer
#pragma unroll
        for (int j = 0; j < STG_COLS / 8; ++j) {
            const int jj = rnd * (STG_COLS / 8) + j, c = 8 * j + cq;
            stg[r0 * STG_PITCH + c] = racc[4 * jj];
            stg[r0 * STG_PITCH + c + 1] = racc[4 * jj + 1];
            stg[(r0 + 8) * STG_PITCH + c] = racc[4 * jj + 2];
            stg[(r0 + 8) * STG_PITCH + c + 1] = racc[4 * jj + 3];
        }
        named_bar_sync(1, kConsumerThreads);
        H3D_SKEW(SKEW_EPILOGUE, 2 * rnd + 1);
        float f[32];
#pragma unroll
        for (int q = 0; q < 32; ++q) f[q] = stg[row * STG_PITCH + half * 32 + q];
        epilogue_store32<PASSES, FP16, SMEM_SCALE>(p, f, pix, n0 + rnd * STG_COLS + half * 32, valid, w_scale);
    }
}

// ------------------------------------------------------------------------------------------ convolution kernel
// Registers per thread after the reallocation at kernel start: __launch_bounds__(384, 1) gives every thread 168, which the BN = 128
// consumers exceed (two fp32 fragments of 64 registers + descriptors: racc spilled to local memory), while the producer warpgroup
// only walks the K loop.  2 * 128 * 232 + 128 * 40 <= 65536.  setmaxnreg.inc only redistributes what the CTA was given at launch, so
// every instance must stay allocated at 168 per thread (ptxas does so for kernels with setmaxnreg; tests/test_build_registers.py).
constexpr int kProducerRegs = 40, kConsumerRegs = 232;

template <int BN, int PASSES, bool FP16>
__global__ void __launch_bounds__(kThreads, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap map_x_hi, const __grid_constant__ CUtensorMap map_x_lo,
               const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo,
               const __grid_constant__ CUtensorMap map_x_h8, const __grid_constant__ CUtensorMap map_w_l8, const TcParams p) {
    // mode 4 operand planes: x_hi = fp16(x), x_lo -> l8 (x residual, e4m3), x_h8 (x, e4m3); w_hi = fp16(w), w_lo -> wh8 (w, e4m3),
    // w_l8 (w residual, e4m3), all pre-scaled so that the three passes fp16 x_hi*w_hi, e4m3 l8*wh8, e4m3 x_h8*w_l8 carry the
    // same power-of-two factor and share one accumulator (split_fmt.cuh); the epilogue multiplies by p.corr_scale.
    using C = RingCfg<BN, PASSES>;
    static_assert(PASSES != 4 || FP16, "fp8-correction mode uses an fp16 main plane");
    static_assert(smem_bytes(BN, PASSES) <= 227 * 1024, "conv_tc_kernel: shared memory budget");

    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    float* stg = reinterpret_cast<float*>(smem + C::STAGES * C::STAGE_BYTES);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::STAGES * C::STAGE_BYTES + STG_BYTES);
    Ring ring{smem, bars, bars + C::STAGES, 0, 0};

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg = __shfl_sync(0xFFFFFFFFu, (int)threadIdx.x / 128, 0);   // warp-uniform role: no divergence around wgmma
    const int kblocks = p.k * p.k * p.cin_chunks;

    if (threadIdx.x == 0) {
        prefetch_tmap(&map_x_hi); prefetch_tmap(&map_w_hi);
        if (PASSES >= 3) { prefetch_tmap(&map_x_lo); prefetch_tmap(&map_w_lo); }
        if (PASSES == 4) { prefetch_tmap(&map_x_h8); prefetch_tmap(&map_w_l8); }
        for (int s = 0; s < C::STAGES; ++s) { mbar_init(&ring.full[s], 1); mbar_init(&ring.empty[s], kConsumerThreads / 32); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    pdl_launch_dependents();
    H3D_SKEW(SKEW_PDL_TAIL, 0);
    pdl_wait();
    const int nb = counted_images(p), num_tiles = counted_tiles(p, nb);   // the producer and the consumers walk the same tiles

    if (wg == 0) {
        setmaxnreg_dec<kProducerRegs>();
        if (warp == 0) {
            // ================================ TMA producer (whole warp, one elected lane issues) ================================
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                const int nt = tile % p.n_tiles, mt = tile / p.n_tiles;
                const int tw = mt % p.tiles_w, th = (mt / p.tiles_w) % p.tiles_h, tb = mt / (p.tiles_w * p.tiles_h);
                const int w0 = tw * p.TW - p.pad, h0 = th * p.TH - p.pad, b0 = tb * p.TB, n0 = nt * BN;
                int kcol = 0;
                for (int kh = 0; kh < p.k; ++kh)
                    for (int kw = 0; kw < p.k; ++kw)
                        for (int cc = 0; cc < p.cin_chunks; ++cc, kcol += BK)
                            produce_kblock<BN, PASSES>(ring, &map_x_hi, &map_x_lo, &map_x_h8, &map_w_hi, &map_w_lo, &map_w_l8, cc * BK,
                                                       w0 + kw, h0 + kh, b0, kcol, n0, p.err_flag);
            }
        }
    } else {
        setmaxnreg_inc<kConsumerRegs>();
        // ================================ wgmma + epilogue (warpgroups 1 and 2) ================================
        const int ct = threadIdx.x - 128;
        float racc[BN / 2];
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            const int nt = tile % p.n_tiles, mt = tile / p.n_tiles;
            const int tw = mt % p.tiles_w, th = (mt / p.tiles_w) % p.tiles_h, tb = mt / (p.tiles_w * p.tiles_h);
            mma_tile<BN, PASSES, FP16>(ring, kblocks, p.chunk_kb, racc, ct >> 7, lane, p.err_flag);
            store_tile<BN, PASSES, FP16>(p, racc, stg, ct, nt * BN, [&](int row, int64_t& pix, bool& valid) {
                const int w_l = row % p.TW, h_l = (row / p.TW) % p.TH, b_l = row / (p.TW * p.TH);
                const int w = tw * p.TW + w_l, h = th * p.TH + h_l, b = tb * p.TB + b_l;
                valid = (w < p.W) && (h < p.H) && (b < nb);
                pix = ((int64_t)b * p.H + h) * p.W + w;
                if (p.pool) {   // 1: pooled output pixel, the even-(w, h) lane of each 2x2 window stores; 2: stride-2 'SAME' conv on an
                                // even-sized map = the stride-1 result at the odd pixels (TF pads 0 before / 1 after, SURVEY.md 9.1)
                    const int par = p.pool == 2 ? 1 : 0;
                    valid = valid && ((w & 1) == par) && ((h & 1) == par);
                    pix = ((int64_t)b * (p.H >> 1) + (h >> 1)) * (p.W >> 1) + (w >> 1);
                }
            }, p.w_scale);
        }
    }
}

// ------------------------------------------------------------------------------------------ first layer (Cin = 3) on tensor cores
// conv1_1 of both networks: 3 -> 64 channels, K = 27.  There is nothing for TMA to fetch (3-channel fp32 pixels), so the A
// operand is BUILT in shared memory: the CTA stages the 18 x 10 x 3 input patch of a 16 x 8 pixel tile, then each of 128 threads
// writes the 27 neighbourhood values of "its" pixel (+ 5 zeros) as hi / lo 16-bit rows in the K-major SWIZZLE_128B layout (rows
// keep the 128-byte pitch of the other kernels, only the first 64 bytes = 32 K values are read).  The 64 x 27 weights are
// converted and stored the same way once per CTA ([W_hi ; W_lo]: 128 rows); fp16 weights with the per-channel shift of
// split_fmt.cuh, whose factors 2^-s the CTA keeps in shared memory for the epilogue.  Per tile each warpgroup runs 2 K steps x 3 passes of
// wgmma (64 pixels x 64 channels) and the shared epilogue.  Two CTAs per SM overlap one CTA's build with the other's stores.
constexpr int C3_TW = 16, C3_TH = 8;
constexpr int C3T_THREADS = 256;
constexpr int C3T_B_BYTES = 128 * BK * 2;
constexpr int C3T_PW = C3_TW + 2, C3T_PH = C3_TH + 2;
constexpr int C3T_PATCH_FLOATS = C3T_PH * C3T_PW * 3;   // 540
constexpr int C3T_SMEM = C3T_B_BYTES + 2 * A_TILE_BYTES + STG_BYTES + C3T_PATCH_FLOATS * 4 + 64 * 4 + 1024 /*align*/;

// COUNTED (p.count set): only images [0, *p.count) are computed, and with slots image b of the launch is image slots[b] of x (the counted
// plan's first layer reads the selected slots in place).  The uncounted instances are the kernel as it was before the count existed.
template <bool FP16, bool COUNTED>
__global__ void __launch_bounds__(C3T_THREADS, 2)
conv_c3_tc_kernel(const float* __restrict__ x, const float* __restrict__ w, const TcParams p, const int* __restrict__ slots) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* bsm = smem;                                   // [W_hi 64 rows ; W_lo 64 rows] x 128 B
    uint8_t* asm_ = smem + C3T_B_BYTES;                    // A_hi | A_lo, 128 rows x 128 B each
    float* stg = reinterpret_cast<float*>(asm_ + 2 * A_TILE_BYTES);
    float* patch = stg + BM * STG_PITCH;                   // [PH][PW][3]
    float* w_scale = patch + C3T_PATCH_FLOATS;             // [64] fp16 weight shifts 2^-s (16-byte aligned)

    const int t = threadIdx.x, wg = t >> 7;
    if (t < 128) {   // weights: row n = output channel (t < 64: hi plane, t >= 64: lo plane of channel t - 64), k = (kh*3 + kw)*3 + ci
        const int co = t & 63;
        int sh = 0;
        if (FP16) {
            float mx = 0.f;
            for (int k = 0; k < 27; ++k) mx = fmaxf(mx, fabsf(__ldg(w + k * 64 + co)));
            sh = fp16_w_shift(mx);
            if (t < 64) w_scale[co] = ldexpf(1.f, -sh);
        }
        uint32_t pk[16];
#pragma unroll
        for (int k2 = 0; k2 < 16; ++k2) {
            float v0 = 0.f, v1 = 0.f;
            if (2 * k2 < 27) v0 = __ldg(w + (2 * k2) * 64 + co);
            if (2 * k2 + 1 < 27) v1 = __ldg(w + (2 * k2 + 1) * 64 + co);
            if (FP16) { v0 = ldexpf(v0, sh); v1 = ldexpf(v1, sh); }
            const uint32_t h = pack_hi2<FP16>(v0, v1);
            if (t < 64) pk[k2] = h;
            else { const float2 r = unpack2<FP16>(h); pk[k2] = pack_hi2<FP16>(v0 - r.x, v1 - r.y); }
        }
#pragma unroll
        for (int c = 0; c < 4; ++c)
            *reinterpret_cast<uint4*>(bsm + sw128_chunk(t, c)) = make_uint4(pk[4 * c], pk[4 * c + 1], pk[4 * c + 2], pk[4 * c + 3]);
    }
    pdl_launch_dependents();
    H3D_SKEW(SKEW_PDL_TAIL, 0);
    pdl_wait();
    const int num_tiles = COUNTED ? counted_tiles(p, counted_images(p)) : p.num_tiles;   // TB = 1: whole images

    const uint32_t sb = smem_u32(bsm), sa = smem_u32(asm_);
    const uint64_t b_hi = desc_sw128(sb), b_lo = desc_sw128(sb + 64 * 128);
    const uint64_t a_hi = desc_sw128(sa + wg * 64 * 128), a_lo = desc_sw128(sa + A_TILE_BYTES + wg * 64 * 128);
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int tw = tile % p.tiles_w, th = (tile / p.tiles_w) % p.tiles_h, b = tile / (p.tiles_w * p.tiles_h);
        {   // haloed input patch, zero outside the image ('SAME' padding)
            const int x0 = tw * C3_TW - 1, y0 = th * C3_TH - 1;
            const float* xb = x + (int64_t)(COUNTED && slots ? slots[b] : b) * p.H * p.W * 3;
            for (int i = t; i < C3T_PATCH_FLOATS; i += C3T_THREADS) {
                const int r = i / (C3T_PW * 3), rem = i - r * (C3T_PW * 3);
                const int gy = y0 + r, gx = x0 + rem / 3;
                float v = 0.f;
                if (gy >= 0 && gy < p.H && gx >= 0 && gx < p.W) v = __ldg(xb + ((int64_t)gy * p.W + x0) * 3 + rem);
                patch[i] = v;
            }
        }
        __syncthreads();   // patch complete; the previous tile's wgmma (waited for) and epilogue reads are done
        if (t < 128) {
            const int w_l = t % C3_TW, h_l = t / C3_TW;
            uint32_t hi[16], lo[16];
#pragma unroll
            for (int k2 = 0; k2 < 16; ++k2) {
                float v0 = 0.f, v1 = 0.f;
                if (2 * k2 < 27) { const int k = 2 * k2; v0 = patch[(h_l + k / 9) * (C3T_PW * 3) + w_l * 3 + (k % 9)]; }
                if (2 * k2 + 1 < 27) { const int k = 2 * k2 + 1; v1 = patch[(h_l + k / 9) * (C3T_PW * 3) + w_l * 3 + (k % 9)]; }
                hi[k2] = pack_hi2<FP16>(v0, v1);
                const float2 r = unpack2<FP16>(hi[k2]);
                lo[k2] = pack_hi2<FP16>(v0 - r.x, v1 - r.y);
            }
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                *reinterpret_cast<uint4*>(asm_ + sw128_chunk(t, c)) = make_uint4(hi[4 * c], hi[4 * c + 1], hi[4 * c + 2], hi[4 * c + 3]);
                *reinterpret_cast<uint4*>(asm_ + A_TILE_BYTES + sw128_chunk(t, c)) = make_uint4(lo[4 * c], lo[4 * c + 1], lo[4 * c + 2], lo[4 * c + 3]);
            }
        }
        fence_proxy_async_smem();      // generic-proxy stores -> visible to the tensor core's async-proxy reads
        __syncthreads();
        float acc[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[i] = 0.f;
        fence_regs<32>(acc);
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < 2; ++j) {                // K = 32 (27 taps x channels + 5 zeros)
            const uint64_t koff = (uint64_t)j * 2;
            mma16<64, FP16>(acc, a_hi + koff, b_hi + koff, (uint32_t)(j != 0));
            mma16<64, FP16>(acc, a_hi + koff, b_lo + koff, 1u);
            mma16<64, FP16>(acc, a_lo + koff, b_hi + koff, 1u);
        }
        wgmma_commit();
        H3D_SKEW(SKEW_COMMIT, tile);
        wgmma_wait<0>();
        fence_regs<32>(acc);
        auto pix_of = [&](int row, int64_t& pix, bool& valid) {
            const int wx = tw * C3_TW + row % C3_TW, hy = th * C3_TH + row / C3_TW;
            valid = (wx < p.W) && (hy < p.H);
            pix = ((int64_t)b * p.H + hy) * p.W + wx;
        };
        if (p.y_lo) store_tile<64, 3, FP16, decltype(pix_of), true>(p, acc, stg, t, 0, pix_of, w_scale);
        else store_tile<64, 1, FP16, decltype(pix_of), true>(p, acc, stg, t, 0, pix_of, w_scale);
    }
}

// ------------------------------------------------------------------------------------------ FC stacks as ONE kernel
// PosePrior (2050 -> 512 -> 512 -> 63, optional 30-wide bottleneck) and ViewpointNet (4098 -> 256 -> 128 -> 3) fully connected stacks
// (nets/ColorHandPose3DNetwork.py:262-267,297-308; nets/PosePriorNetwork.py:113-116) followed by Rodrigues / flip / rotate
// (:239-247,311-361) in a single launch instead of one launch per layer + the rotation kernel.
//  * A fully connected layer is the 1x1 case of the implicit GEMM above: M = 128 batch rows (TMA zero-fills rows >= B), N = 64 output
//    features per tile, K = in_features in blocks of 64, 3-pass wgmma.
//  * One CLUSTER of 8 CTAs per chain: CTA r of the cluster owns the N tiles r, r + 8, ... of every layer, so the 4.2 MB weight matrix of
//    the first layer streams through 8 SMs.  Hidden activations go through global memory (L2-resident, <= 128 KB) as split planes;
//    between layers every thread fences (generic -> async proxy, the next layer reads through TMA) and the cluster synchronises.
//  * The shared-memory ring and its barrier phases simply continue across layers (a layer is a tile loop).
//  * Two chains = two clusters in the same grid.  The cluster that finishes LAST (atomic ticket at device scope) applies the
//    Rodrigues / flip / rotate epilogue to the canonical coordinates and the view-point vector of both chains.
constexpr int kFcMaxLayers = 4;
constexpr int kFcCluster = 8;
struct FcLayer {
    CUtensorMap map_x_hi, map_x_lo, map_w_hi, map_w_lo;
    TcParams p;            // epilogue parameters (bias, outputs, n_valid, leaky); B / geometry fields unused
    int kblocks, m_tiles, n_tiles, pad_;
};
struct FcChain { FcLayer layer[kFcMaxLayers]; int num_layers; int pad_[3]; };
struct FcChainParams {
    FcChain chain[2];
    int num_chains, B;
    const float* can; const float* uxyz; const float* hand_side;   // rotate epilogue (num_chains == 2)
    float* rot; float* out;
    unsigned int* counter;
    int* err_flag;
};

__device__ __forceinline__ void fc_layer_sync(int l) {
    __threadfence();                                        // the layer's outputs: visible at device scope ...
    asm volatile("fence.proxy.async;" ::: "memory");        // ... and to the async proxy (the next layer's TMA loads)
    H3D_SKEW(SKEW_CLUSTER, l);
    cluster_sync_all();
}

template <bool FP16>
__global__ void __cluster_dims__(kFcCluster, 1, 1) __launch_bounds__(kThreads, 1)
fc_chain_kernel(const __grid_constant__ FcChainParams P) {
    constexpr int BN = 64, PASSES = 3;
    constexpr int kChunk = 9;                              // K blocks per tensor-core partial sum (as the convolution kernels)
    using C = RingCfg<BN, PASSES>;

    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    float* stg = reinterpret_cast<float*>(smem + C::STAGES * C::STAGE_BYTES);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::STAGES * C::STAGE_BYTES + STG_BYTES);
    Ring ring{smem, bars, bars + C::STAGES, 0, 0};
    int& s_last = *reinterpret_cast<int*>(bars + 2 * C::STAGES);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int rank = (int)cluster_ctarank();
    const int wg = __shfl_sync(0xFFFFFFFFu, (int)threadIdx.x / 128, 0);
    const FcChain& ch = P.chain[blockIdx.x / kFcCluster];

    if (threadIdx.x == 0) {
        for (int l = 0; l < ch.num_layers; ++l) {
            prefetch_tmap(&ch.layer[l].map_x_hi); prefetch_tmap(&ch.layer[l].map_x_lo);
            prefetch_tmap(&ch.layer[l].map_w_hi); prefetch_tmap(&ch.layer[l].map_w_lo);
        }
        for (int s = 0; s < C::STAGES; ++s) { mbar_init(&ring.full[s], 1); mbar_init(&ring.empty[s], kConsumerThreads / 32); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    pdl_launch_dependents();
    H3D_SKEW(SKEW_PDL_TAIL, 0);
    pdl_wait();

    // Every warp of every CTA of the cluster runs the SAME layer loop and reaches fc_layer_sync() exactly once per layer.
    for (int l = 0; l < ch.num_layers; ++l) {
        const FcLayer& L = ch.layer[l];
        const int items = L.m_tiles * L.n_tiles;
        if (warp == 0) {
            for (int item = rank; item < items; item += kFcCluster) {
                const int nt = item % L.n_tiles, mt = item / L.n_tiles;
                for (int kb = 0; kb < L.kblocks; ++kb)
                    produce_kblock<BN, PASSES>(ring, &L.map_x_hi, &L.map_x_lo, &L.map_x_hi, &L.map_w_hi, &L.map_w_lo, &L.map_w_hi, kb * BK, 0, 0,
                                               mt * BM, kb * BK, nt * BN, P.err_flag);
            }
        } else if (wg >= 1) {
            const int ct = threadIdx.x - 128;
            float racc[BN / 2];
            for (int item = rank; item < items; item += kFcCluster) {
                const int nt = item % L.n_tiles, mt = item / L.n_tiles;
                mma_tile<BN, PASSES, FP16>(ring, L.kblocks, kChunk, racc, ct >> 7, lane, P.err_flag);
                store_tile<BN, PASSES, FP16>(L.p, racc, stg, ct, nt * BN, [&](int row, int64_t& pix, bool& valid) {
                    pix = (int64_t)mt * BM + row;
                    valid = pix < P.B;
                }, L.p.w_scale);
            }
        }
        fc_layer_sync(l);
    }

    // ---- last cluster to finish: Rodrigues + right-hand flip + rotation of the canonical coordinates (both chains' outputs)
    if (P.num_chains == 2 && rank == 0) {
        H3D_SKEW(SKEW_TICKET, 0);
        if (threadIdx.x == 0) {
            __threadfence();
            s_last = atomicAdd(P.counter, 1u) == 1u;
            if (s_last) *P.counter = 0u;                    // ready for the next launch (launches are stream ordered)
        }
        __syncthreads();
        if (s_last) {
            __threadfence();
            for (int b = warp; b < P.B; b += kThreads / 32) {
                float R[9];
                if (lane == 0) rodrigues_rot_mat(__ldcg(P.uxyz + 3 * b), __ldcg(P.uxyz + 3 * b + 1), __ldcg(P.uxyz + 3 * b + 2), R);
#pragma unroll
                for (int i = 0; i < 9; ++i) R[i] = __shfl_sync(0xFFFFFFFFu, R[i], 0);
                if (P.rot && lane < 9) P.rot[9 * b + lane] = R[lane];
                const bool right = P.hand_side[2 * b + 1] > P.hand_side[2 * b];
                for (int i = lane; i < 63; i += 32) {
                    float c3[3];
                    const int kp = i / 3;
                    c3[0] = __ldcg(P.can + 63 * b + 3 * kp); c3[1] = __ldcg(P.can + 63 * b + 3 * kp + 1); c3[2] = __ldcg(P.can + 63 * b + 3 * kp + 2);
                    const int j = i - kp * 3;
                    const float cz = right ? -c3[2] : c3[2];
                    P.out[63 * b + i] = c3[0] * R[j] + c3[1] * R[3 + j] + cz * R[6 + j];
                }
            }
        }
    }
    H3D_SKEW(SKEW_CLUSTER, ch.num_layers);
    cluster_sync_all();          // no CTA of the cluster exits while a peer may still be inside a cluster barrier
}

}  // namespace

// ------------------------------------------------------------------------------------------ host
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (fn) return fn;
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !ptr) {
        set_error("cuTensorMapEncodeTiled not available (%s)", cudaGetErrorString(e));
        return nullptr;
    }
    fn = reinterpret_cast<EncodeTiledFn>(ptr);
    return fn;
}

// es = element size in bytes: 2 (bf16 / fp16 planes, 128-byte rows, SWIZZLE_128B) or 1 (e4m3 planes, 64-byte rows, SWIZZLE_64B)
bool encode_act_map(CUtensorMap* m, const void* base, int C_total, int C_used, int W, int H, int B, int TW, int TH, int TB, int es) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return false;
    cuuint64_t dims[4] = {(cuuint64_t)C_used, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)C_total * es, (cuuint64_t)W * C_total * es, (cuuint64_t)H * W * C_total * es};
    cuuint32_t box[4] = {(cuuint32_t)BK, (cuuint32_t)TW, (cuuint32_t)TH, (cuuint32_t)TB};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = fn(m, es == 2 ? CU_TENSOR_MAP_DATA_TYPE_UINT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, const_cast<void*>(base), dims, strides,
                    box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, es == 2 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(activations) failed: %d", (int)r); return false; }
    return true;
}

bool encode_w_map(CUtensorMap* m, const void* base, int Ktot, int Cout_pad, int BN, int es) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return false;
    cuuint64_t dims[2] = {(cuuint64_t)Ktot, (cuuint64_t)Cout_pad};
    cuuint64_t strides[1] = {(cuuint64_t)Ktot * es};
    cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)BN};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(m, es == 2 ? CU_TENSOR_MAP_DATA_TYPE_UINT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), dims, strides,
                    box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, es == 2 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(weights) failed: %d", (int)r); return false; }
    return true;
}

namespace {

void choose_tile(int B, int H, int W, int* TW, int* TH, int* TB, bool pool = false) {
    static const int cand[][3] = {{16, 8, 1}, {8, 16, 1}, {32, 4, 1}, {4, 32, 1}, {64, 2, 1}, {128, 1, 1}, {8, 8, 2},
                                  {16, 4, 2}, {4, 16, 2}, {8, 4, 4}, {4, 8, 4}, {4, 4, 8}, {8, 2, 8}, {2, 2, 32}, {1, 1, 128}};
    int64_t best = -1;
    for (auto& c : cand) {
        if (pool && !((c[0] % 2) == 0 && c[0] <= 16 && (c[1] % 2) == 0)) continue;   // 2x2 windows must stay inside one warp
        const int64_t tiles = (int64_t)ceil_div(W, c[0]) * ceil_div(H, c[1]) * ceil_div(B, c[2]);
        if (best < 0 || tiles < best) { best = tiles; *TW = c[0]; *TH = c[1]; *TB = c[2]; }
    }
}

template <int BN, int PASSES, bool FP16>
int launch_inst(const TcConvPlan* pl, cudaStream_t s);

}  // namespace

struct TcConvPlan {
    int device = 0;
    TcConvDesc d;
    CUtensorMap map_x_hi, map_x_lo, map_w_hi, map_w_lo, map_x_h8, map_w_l8;
    TcParams p;
    int BN, grid;
};

// SM count and the shared-memory opt-in are per DEVICE (one process may hold contexts on several GPUs)
constexpr int kMaxDevices = 64;
static int current_device() { int dev = 0; if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); dev = 0; } return dev; }
int tc_num_sms() {
    static int n[kMaxDevices] = {};
    const int dev = current_device() % kMaxDevices;
    if (!n[dev]) {
        int v = 0;
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) { cudaGetLastError(); v = 132; }
        n[dev] = v;
    }
    return n[dev];
}
// once per (kernel instance, device): raise the dynamic shared-memory limit
template <typename K>
static int smem_opt_in(K kernel, int bytes, bool* done /*[kMaxDevices]*/) {
    const int dev = current_device() % kMaxDevices;
    if (!done[dev]) {
        H3D_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        done[dev] = true;
    }
    return H3D_OK;
}

// Launch with the programmatic-stream-serialization attribute (see pdl_wait above); tune.pdl = 0 gives plain stream order.
template <typename... KArgs, typename... Args>
static cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = tc_tuning().pdl ? 1 : 0;
    cfg.attrs = attr; cfg.numAttrs = 1;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
    if (e == cudaSuccess) ++t_launches;   // as H3D_CHECK_LAUNCH
    return e;
}

// Tuning switches (A/B experiments, forced variants in the tests).  Read from the environment ONCE, when the library is first
// used, and changeable afterwards only through tc_set_tuning() (h3d_set_tuning): nothing on a launch path calls getenv.
TcTuning& tc_tuning() {
    static TcTuning t = [] {
        TcTuning v;
        auto geti = [](const char* n, int d) { const char* e = getenv(n); return e ? atoi(e) : d; };
        v.bn = geti("H3D_TC_BN", 0);
        v.chunk_kb = geti("H3D_TC_CHUNK_KB", 0);
        v.no_side_stream = geti("H3D_NO_SIDE_STREAM", 0);
        v.no_pool_fusion = geti("H3D_NO_POOL_FUSION", 0);
        v.lift_direct = geti("H3D_LIFT_DIRECT", 0);
        v.c3_ffma = geti("H3D_C3_FFMA", 0);
        v.pdl = geti("H3D_PDL", 1);
        v.fc_chain = geti("H3D_FC_CHAIN", 1);
        v.no_seg_fusion = geti("H3D_NO_SEG_FUSION", 0);
        return v;
    }();
    return t;
}
#ifdef H3D_SKEW_BUILD
// Schedule-skew config (skew.cuh): the host copy and the uploaders of every translation unit with hooks.
static std::vector<int (*)(const SkewCfg&)>& skew_uploaders() { static std::vector<int (*)(const SkewCfg&)> v; return v; }
static SkewCfg g_skew_host = {};
int skew_register(int (*upload)(const SkewCfg&)) { skew_uploaders().push_back(upload); return 0; }
int skew_set(const char* key, int value) {
    static const char* const sites[SKEW_SITES] = {"producer", "consumer", "commit", "epilogue", "cluster", "pdl_tail", "ticket"};
    const std::string k(key);
    if (k == "skew_reset") g_skew_host = SkewCfg{};
    else {
        int s = 0;
        while (s < SKEW_SITES && k.compare(0, 5 + strlen(sites[s]) + 1, std::string("skew_") + sites[s] + "_") != 0) ++s;
        const std::string f = s < SKEW_SITES ? k.substr(5 + strlen(sites[s]) + 1) : "";
        SkewSiteCfg* c = s < SKEW_SITES ? &g_skew_host.site[s] : nullptr;
        if (c && f == "ns" && value >= 0) c->ns = std::min((unsigned)value, kSkewMaxNs);
        else if (c && f == "role" && value >= 0 && value <= SKEW_RANK0 + 15) c->role = (unsigned)value;
        else if (c && f == "period" && value >= 0) c->period = (unsigned)value;
        else if (c && f == "seed") c->seed = (unsigned)value;
        else { set_error("h3d_set_tuning: bad skew key '%s' or value %d", key, value); return H3D_EINVAL; }
    }
    for (auto up : skew_uploaders()) H3D_CUDA((cudaError_t)up(g_skew_host));
    return H3D_OK;
}
#endif

int tc_set_tuning(const char* key, int value) {
    TcTuning& t = tc_tuning();
    const std::string k(key ? key : "");
    if (k == "tc_bn") t.bn = value;
    else if (k == "tc_chunk_kb") t.chunk_kb = value;
    else if (k == "no_side_stream") t.no_side_stream = value;
    else if (k == "no_pool_fusion") t.no_pool_fusion = value;
    else if (k == "lift_direct") t.lift_direct = value;
    else if (k == "c3_ffma") t.c3_ffma = value;
    else if (k == "pdl") t.pdl = value;
    else if (k == "fc_chain") t.fc_chain = value;
    else if (k == "no_seg_fusion") t.no_seg_fusion = value;
#ifdef H3D_SKEW_BUILD
    else if (k.compare(0, 5, "skew_") == 0) return skew_set(key, value);
#endif
    else { set_error("h3d_set_tuning: unknown key '%s'", k.c_str()); return H3D_EINVAL; }
    return H3D_OK;
}

namespace {
// N = 128 tiles where Cout allows (each A tile feeds twice the output channels).  Small maps (lifting pyramids from 16x16
// down, 1x1 layers over batch rows) have too few pixel tiles to fill the machine with wide tiles, so N = 64 tiles spread the
// work over twice the SMs.  The rule depends on the layer geometry only, never on the batch size: the arithmetic of an image
// must not depend on how a batch is cut (tests/test_gpu_properties.py: bit-identical results under sharding).
int choose_bn(int H, int W, int Cout_pad, int passes) {
    const TcTuning& tune = tc_tuning();
    int BN = Cout_pad % 128 == 0 ? 128 : 64;
    if ((int64_t)H * W <= 256) BN = 64;
    if ((tune.bn == 64 || tune.bn == 128) && Cout_pad % tune.bn == 0) BN = tune.bn;
    if (passes == 4) BN = 64;   // the separate e4m3 accumulator: three fragments of BN / 2 registers per thread
    return BN;
}

template <int BN, int PASSES, bool FP16>
int launch_inst(const TcConvPlan* pl, cudaStream_t s) {
    constexpr int smem = smem_bytes(BN, PASSES);
    static bool attr[kMaxDevices] = {};
    if (int rc = smem_opt_in(conv_tc_kernel<BN, PASSES, FP16>, smem, attr)) return rc;
    H3D_CUDA(launch_pdl(conv_tc_kernel<BN, PASSES, FP16>, dim3(pl->grid), dim3(kThreads), smem, s, pl->map_x_hi, pl->map_x_lo, pl->map_w_hi,
                        pl->map_w_lo, pl->map_x_h8, pl->map_w_l8, pl->p));
    return H3D_OK;
}
}  // namespace

TcConvPlan* tc_conv_plan_create(const TcConvDesc& d, int* rc) {
    int rc_local;
    if (!rc) rc = &rc_local;
    *rc = H3D_EINVAL;   // every early return below is an illegal descriptor
    if (d.Cin_pad % BK != 0 || d.Cout_pad % 64 != 0 || (d.k != 1 && d.k != 3 && d.k != 5 && d.k != 7) || (d.passes != 1 && d.passes != 3 && d.passes != 4)) {
        set_error("tc_conv: unsupported geometry (Cin_pad=%d Cout_pad=%d k=%d passes=%d)", d.Cin_pad, d.Cout_pad, d.k, d.passes);
        return nullptr;
    }
    const bool padded_out = d.Cout % 32 != 0;   // masked scalar tail in the epilogue: no alignment requirement there
    if (d.y.hi && ((d.Cy_total % 8) || (d.cy_off % 8))) { set_error("tc_conv: split output channel offset/stride must be multiples of 8"); return nullptr; }
    if (d.yf && !padded_out && ((d.Cyf_total % 4) || (d.cyf_off % 4))) { set_error("tc_conv: fp32 output channel offset/stride must be multiples of 4"); return nullptr; }
    if (padded_out && d.pool == 1) { set_error("tc_conv: fused pooling needs Cout %% 32 == 0"); return nullptr; }
    if (d.pool < 0 || d.pool > 2) { set_error("tc_conv: pool mode must be 0 (none), 1 (max-pool) or 2 (stride 2)"); return nullptr; }
    if (d.pool == 2 && d.k < 3) { set_error("tc_conv: stride 2 needs k >= 3 (for k = 1 TF's 'SAME' samples the even pixels, not the odd ones)"); return nullptr; }
    if (d.passes == 3 && (!d.x.lo || !d.w.lo)) { set_error("tc_conv: 3-pass mode needs lo planes"); return nullptr; }
    if (d.passes == 4 && (!d.x.l8 || !d.x.h8 || !d.w.l8 || !d.w.h8 || d.half != Half16::FP16 || d.corr_scale <= 0.f)) {
        set_error("tc_conv: fp8-correction mode needs fp16 + e4m3 l8/h8 planes for activations and weights and a correction scale");
        return nullptr;
    }
    if (d.half == Half16::FP16 && d.passes != 4 && !d.w_scale) { set_error("tc_conv: fp16 weight planes need their per-channel scales"); return nullptr; }
    if (d.passes == 4 && d.y.hi && (!d.y.l8 || !d.y.h8)) { set_error("tc_conv: fp8-correction mode needs l8/h8 output planes"); return nullptr; }
    if (d.passes == 4 && d.y.hi && ((d.Cy_total % 16) || (d.cy_off % 16))) { set_error("tc_conv: fp8 planes need 16-channel aligned offsets"); return nullptr; }
    if (d.pool && ((d.H | d.W) & 1)) { set_error("tc_conv: fused max-pool / stride 2 needs even H and W"); return nullptr; }
    *rc = H3D_ECUDA;    // from here on only a tensor-map encode can fail
    TcConvPlan* pl = new TcConvPlan();
    pl->d = d;
    const TcTuning& tune = tc_tuning();
    const int BN = choose_bn(d.H, d.W, d.Cout_pad, d.passes);
    int TW, TH, TB;
    choose_tile(d.B, d.H, d.W, &TW, &TH, &TB, d.pool == 1);
    pl->BN = BN;
    pl->device = current_device();
    TcParams& p = pl->p;
    p.bias = d.bias;
    p.y_hi = d.y.hi; p.y_lo = d.y.lo; p.y_l8 = d.y.l8; p.y_h8 = d.y.h8; p.Cy_total = d.Cy_total; p.cy_off = d.cy_off;
    p.corr_scale = d.corr_scale;
    p.yf = d.yf; p.Cyf_total = d.Cyf_total; p.cyf_off = d.cyf_off;
    p.B = d.B; p.H = d.H; p.W = d.W; p.k = d.k; p.pad = d.k / 2; p.cin_chunks = d.Cin_pad / BK;
    p.TW = TW; p.TH = TH; p.TB = TB;
    p.tiles_w = ceil_div(d.W, TW); p.tiles_h = ceil_div(d.H, TH);
    p.n_tiles = d.Cout_pad / BN;
    p.num_tiles = p.tiles_w * p.tiles_h * ceil_div(d.B, TB) * p.n_tiles;
    p.leaky = d.leaky;
    p.n_valid = d.Cout;
    p.pool = d.pool;
    p.err_flag = d.err_flag;
    p.w_scale = d.w_scale;
    p.count = d.count;
    // <= ~108 accumulating tensor-core steps per partial sum (9 K blocks x 4 K steps x 3 passes)
    p.chunk_kb = d.passes >= 3 ? 9 : 27;
    if (tune.chunk_kb > 0) p.chunk_kb = tune.chunk_kb;
    pl->grid = std::min(p.num_tiles, tc_num_sms());
    const int Ktot = d.k * d.k * d.Cin_pad;
    bool ok = encode_act_map(&pl->map_x_hi, d.x.hi, d.Cin_total, d.Cin_pad, d.W, d.H, d.B, TW, TH, TB) &&
              encode_w_map(&pl->map_w_hi, d.w.hi, Ktot, d.Cout_pad, BN);
    if (ok && d.passes == 3)
        ok = encode_act_map(&pl->map_x_lo, d.x.lo, d.Cin_total, d.Cin_pad, d.W, d.H, d.B, TW, TH, TB) &&
             encode_w_map(&pl->map_w_lo, d.w.lo, Ktot, d.Cout_pad, BN);
    if (ok && d.passes == 4)   // e4m3 planes: x residual (slot "lo"), x coarse, w coarse (slot "lo"), w residual
        ok = encode_act_map(&pl->map_x_lo, d.x.l8, d.Cin_total, d.Cin_pad, d.W, d.H, d.B, TW, TH, TB, 1) &&
             encode_act_map(&pl->map_x_h8, d.x.h8, d.Cin_total, d.Cin_pad, d.W, d.H, d.B, TW, TH, TB, 1) &&
             encode_w_map(&pl->map_w_lo, d.w.h8, Ktot, d.Cout_pad, BN, 1) &&
             encode_w_map(&pl->map_w_l8, d.w.l8, Ktot, d.Cout_pad, BN, 1);
    if (ok && d.passes == 1) { pl->map_x_lo = pl->map_x_hi; pl->map_w_lo = pl->map_w_hi; }
    if (ok && d.passes != 4) { pl->map_x_h8 = pl->map_x_hi; pl->map_w_l8 = pl->map_w_hi; }
    if (!ok) { delete pl; return nullptr; }
    *rc = H3D_OK;
    return pl;
}

void tc_conv_plan_destroy(TcConvPlan* p) { delete p; }

void tc_conv_geometry(int B, int H, int W, int Cout_pad, int pool, int passes, int out[4]) {
    choose_tile(B, H, W, &out[0], &out[1], &out[2], pool == 1);
    out[3] = choose_bn(H, W, Cout_pad, passes);
}

int64_t tc_conv_flops(const TcConvPlan* p) {
    return 2ll * p->d.B * p->d.H * p->d.W * p->d.k * p->d.k * (int64_t)p->d.Cin_pad * p->d.Cout_pad;
}

int tc_conv_launch(const TcConvPlan* pl, cudaStream_t s) {
    const bool fp16 = pl->d.half == Half16::FP16;
    const int key = pl->BN * 10 + pl->d.passes;
#define CASE(BN_, P_)                                                                  \
    case BN_ * 10 + P_:                                                                \
        return fp16 ? launch_inst<BN_, P_, true>(pl, s) : launch_inst<BN_, P_, false>(pl, s);
    switch (key) {
        CASE(64, 1) CASE(64, 3) CASE(128, 1) CASE(128, 3)
        case 64 * 10 + 4: return launch_inst<64, 4, true>(pl, s);      // fp16 + e4m3 corrections
    }
#undef CASE
    set_error("tc_conv: no kernel instance for BN=%d passes=%d", pl->BN, pl->d.passes);
    return H3D_EINVAL;
}

// conv1_1 (3 -> 64 channels, 3x3, stride 1) on the tensor cores: x fp32 [B,H,W,3], w fp32 HWIO [3,3,3,64] and bias [64] on the
// device, output split planes y (hi, and lo when present) [B,H,W,Cs_total] at channel offset cs_off.
int launch_conv_c3_tc(const float* x, const float* w, const float* bias, Split y, int Cs_total, int cs_off, int B, int H, int W, int leaky,
                      Half16 half, cudaStream_t s, int* err_flag, const int* count, const int* slots) {
    H3D_REQUIRE(x && w && bias && y.hi && !y.l8 && (Cs_total % 8) == 0 && (cs_off % 8) == 0, "conv_c3_tc: bad argument");
    TcParams p{};
    p.bias = bias;
    p.y_hi = y.hi; p.y_lo = y.lo; p.Cy_total = Cs_total; p.cy_off = cs_off;
    p.corr_scale = 1.f;
    p.B = B; p.H = H; p.W = W; p.k = 3; p.pad = 1; p.cin_chunks = 1;
    p.TW = C3_TW; p.TH = C3_TH; p.TB = 1;
    p.tiles_w = ceil_div(W, C3_TW); p.tiles_h = ceil_div(H, C3_TH); p.n_tiles = 1;
    p.num_tiles = p.tiles_w * p.tiles_h * B;
    p.n_valid = 64; p.pool = 0; p.chunk_kb = 1; p.leaky = leaky; p.err_flag = err_flag; p.count = count;
    const int grid = std::min(p.num_tiles, 2 * tc_num_sms());   // two co-resident CTAs per SM
    static bool attr[4][kMaxDevices] = {};
    if (int rc = smem_opt_in(conv_c3_tc_kernel<true, false>, C3T_SMEM, attr[0])) return rc;
    if (int rc = smem_opt_in(conv_c3_tc_kernel<false, false>, C3T_SMEM, attr[1])) return rc;
    if (int rc = smem_opt_in(conv_c3_tc_kernel<true, true>, C3T_SMEM, attr[2])) return rc;
    if (int rc = smem_opt_in(conv_c3_tc_kernel<false, true>, C3T_SMEM, attr[3])) return rc;
    auto* k = half == Half16::FP16 ? (count ? conv_c3_tc_kernel<true, true> : conv_c3_tc_kernel<true, false>)
                                   : (count ? conv_c3_tc_kernel<false, true> : conv_c3_tc_kernel<false, false>);
    H3D_CUDA(launch_pdl(k, dim3(grid), dim3(C3T_THREADS), (size_t)C3T_SMEM, s, x, w, p, slots));
    return H3D_OK;
}

// ------------------------------------------------------------------------------------------ FC chain: host
struct FcChainPlan { FcChainParams P; Half16 half; int grid; };

FcChainPlan* fc_chain_plan_create(const FcChainDesc* chains, int num_chains, int B, Half16 half, const float* can, const float* uxyz,
                                  unsigned int* counter, int* err_flag) {
    if (num_chains < 1 || num_chains > 2 || B < 1) { set_error("fc_chain: bad geometry"); return nullptr; }
    FcChainPlan* pl = new FcChainPlan();
    memset(&pl->P, 0, sizeof(pl->P));
    pl->half = half; pl->grid = num_chains * kFcCluster;
    FcChainParams& P = pl->P;
    P.num_chains = num_chains; P.B = B; P.can = can; P.uxyz = uxyz; P.counter = counter; P.err_flag = err_flag;
    for (int c = 0; c < num_chains; ++c) {
        const FcChainDesc& cd = chains[c];
        if (cd.num_layers < 1 || cd.num_layers > kFcMaxLayers) { set_error("fc_chain: 1..4 layers per chain"); delete pl; return nullptr; }
        P.chain[c].num_layers = cd.num_layers;
        for (int l = 0; l < cd.num_layers; ++l) {
            const FcLayerDesc& d = cd.layer[l];
            FcLayer& L = P.chain[c].layer[l];
            const int Kpad = (int)align_up(d.in_features, BK);
            if (!d.x.hi || !d.x.lo || !d.w.hi || !d.w.lo || d.out_pad % 64 || d.x_stride < Kpad || (d.y.hi && (d.y_stride % 8)) ||
                (half == Half16::FP16 && !d.w_scale)) {
                set_error("fc_chain: bad layer %d of chain %d", l, c); delete pl; return nullptr;
            }
            bool ok = encode_act_map(&L.map_x_hi, d.x.hi, d.x_stride, Kpad, 1, 1, B, 1, 1, BM) &&
                      encode_act_map(&L.map_x_lo, d.x.lo, d.x_stride, Kpad, 1, 1, B, 1, 1, BM) &&
                      encode_w_map(&L.map_w_hi, d.w.hi, Kpad, d.out_pad, 64) && encode_w_map(&L.map_w_lo, d.w.lo, Kpad, d.out_pad, 64);
            if (!ok) { delete pl; return nullptr; }
            L.kblocks = Kpad / BK; L.m_tiles = ceil_div(B, BM); L.n_tiles = d.out_pad / 64;
            TcParams& p = L.p;
            p.bias = d.bias; p.y_hi = d.y.hi; p.y_lo = d.y.lo; p.Cy_total = d.y_stride; p.cy_off = 0; p.corr_scale = 1.f;
            p.yf = d.yf; p.Cyf_total = d.yf_stride; p.cyf_off = 0;
            p.B = B; p.H = 1; p.W = 1; p.k = 1; p.TW = 1; p.TH = 1; p.TB = BM;
            p.n_valid = d.out_features; p.pool = 0; p.leaky = d.leaky; p.err_flag = err_flag; p.w_scale = d.w_scale;
        }
    }
    return pl;
}

void fc_chain_plan_destroy(FcChainPlan* p) { delete p; }

int fc_chain_launch(const FcChainPlan* pl, const float* hand_side, float* rot, float* out, cudaStream_t s) {
    FcChainParams P = pl->P;
    P.hand_side = hand_side; P.rot = rot; P.out = out;
    H3D_REQUIRE(P.num_chains == 1 || (hand_side && out), "fc_chain: hand_side / out are required for the rotation epilogue");
    constexpr int smem = smem_bytes(64, 3);
    static bool at_h[kMaxDevices] = {}, at_b[kMaxDevices] = {};
    if (pl->half == Half16::FP16) {
        if (int rc = smem_opt_in(fc_chain_kernel<true>, smem, at_h)) return rc;
        H3D_CUDA(launch_pdl(fc_chain_kernel<true>, dim3(pl->grid), dim3(kThreads), (size_t)smem, s, P));
    } else {
        if (int rc = smem_opt_in(fc_chain_kernel<false>, smem, at_b)) return rc;
        H3D_CUDA(launch_pdl(fc_chain_kernel<false>, dim3(pl->grid), dim3(kThreads), (size_t)smem, s, P));
    }
    return H3D_OK;
}

}  // namespace h3d

// Backward of the tensor-core convolution y = act(conv_SAME(x, w, stride) + b) (conv_wgmma.cu, utils/general.py:36-59), the
// gradients TF's Conv2DBackpropInput / Conv2DBackpropFilter / BiasAddGrad / Maximum-gradient compute under AdamOptimizer.minimize
// (training_posenet.py:67, training_handsegnet.py).
//
// * Gradient prep (one HBM pass): dy' = dy * act'(y) (1 where y >= 0, 0.01 elsewhere) as split planes [B,H,W,Cout_pad] at the
//   INPUT resolution.  A stride-2 layer is the stride-1 'SAME' result at the odd pixels, so its adjoint scatters dy' to the odd
//   pixels of a zero map and continues as a stride-1 adjoint.  Per-block fixed-order column sums of dy' give the bias gradient.
// * Data gradient: dx = conv_SAME(dy', W_d) with W_d[ci][kh][kw][co] = w[k-1-kh][k-1-kw][ci][co] (odd k, symmetric padding), run
//   by the forward kernel (tc_conv_plan_create) on planes packed on the device by pack_conv_w_kernel.
// * Weight gradient (conv_wgrad_tc_kernel): for each tap t = (kh, kw), dW_t[co, ci] = sum_p dy'[p, co] x[p + t - pad, ci], a GEMM
//   with M = Cout, N = Cin and K = pixels.  Both operands are the 4-D activation boxes {64 ch, TW, TH, TB} of the forward (64 pixel
//   rows x 128 bytes): the dy' box at the pixel tile, the x box at the tile shifted by the tap, TMA's zero fill supplying the 'SAME'
//   padding and the ragged tile edges.  In shared memory a box is the MN-major SWIZZLE_128B layout (channels contiguous), so
//   both operands go to wgmma with the transpose bits set.  A CTA owns one (tap, 64 Cout, BN Cin) tile and one contiguous range
//   of pixel blocks (split-K); its two consumer warpgroups take alternate pixel blocks, each folds its tensor-core partial sums
//   into fp32 registers every chunk_kb blocks, and the epilogue adds warpgroup 2's fragment to warpgroup 1's and stores the
//   tile.  wgrad_reduce_kernel sums the splits in a fixed order into HWIO dW: the result is bit-reproducible run to run.
#include <cuda.h>

#include <algorithm>

#include "common.cuh"
#include "split_fmt.cuh"
#include "wgmma_common.cuh"

namespace h3d {

namespace {

constexpr int WG_ROWS = 64;                          // pixels per K block (one TMA box)
constexpr int WG_BOX_BYTES = WG_ROWS * 128;          // one box of 64 channels x 64 pixels, 16-bit
constexpr int kWgThreads = 384;                      // warpgroup 0: TMA producer, warpgroups 1-2: wgmma
constexpr int kWgSmemBudget = 227 * 1024 - 2048;     // ring stages; 2 KB: alignment slack + barriers
constexpr int kWgProducerRegs = 40, kWgConsumerRegs = 232;   // as conv_tc_kernel: 2 * 128 * 232 + 128 * 40 <= 65536

// stage = [dy' hi | dy' lo | x hi (BN / 64 boxes) | x lo (BN / 64 boxes)]; PASSES 1 drops the lo planes
__host__ __device__ constexpr int wg_stage_bytes(int BN, int PASSES) { return (PASSES == 3 ? 2 : 1) * (1 + BN / 64) * WG_BOX_BYTES; }
// An even count, at most 8.  Warpgroup cw consumes the K blocks kb = cw, cw + 2, ... from stage kb % STAGES, so with an even count
// each stage has one consumer, which has taken round r - 1 of its full barrier before it waits for round r.  With an odd count (7 at
// BN = 64 in 3 passes) the two warpgroups alternate on a stage: one could wait for round r while the other's round r - 1 had not
// landed, and the parity wait would pass at once on the stage's old contents.
__host__ __device__ constexpr int wg_num_stages(int BN, int PASSES) {
    return (kWgSmemBudget / wg_stage_bytes(BN, PASSES) > 8 ? 8 : kWgSmemBudget / wg_stage_bytes(BN, PASSES)) & ~1;
}
__host__ __device__ constexpr int wg_smem_bytes(int BN, int PASSES) { return wg_num_stages(BN, PASSES) * wg_stage_bytes(BN, PASSES) + 2048; }

struct WgradParams {
    float* partial;      // [splits][num_tiles][BN][64] fp32: element (ci, co) of every CTA's tile
    int k, pad, m_tiles, n_tiles, num_tiles, splits;
    int TW, TH, TB, tiles_w, tiles_h, pix_blocks;
    int chunk_kb;        // K blocks (per warpgroup) accumulated inside the tensor core before the fold into fp32 registers
    int* err_flag;
};

// MN-major SWIZZLE_128B matrix descriptor: rows of 128 bytes hold 64 consecutive M (or N) elements, groups of 8 rows (1024-byte atoms)
// follow each other along K at the stride byte offset (bits 32-45), and further 64-element M / N blocks sit at the leading byte offset
// (bits 16-29).  The roles of the two offsets are those of the K-major desc_sw128 exchanged.
__device__ __forceinline__ uint64_t desc_mn_sw128(uint32_t saddr, uint32_t lbo_bytes) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) | (64ull << 32) | (1ull << 62);
}

// D[64 x N] (+)= A[64 x 16] B[16 x N], bf16 operands, both MN-major in shared memory (imm-trans-a = imm-trans-b = 1)
__device__ __forceinline__ void wgmma_bf16_n64_tt(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_bf16_n128_tt(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(scale_d));
}
template <int N>
__device__ __forceinline__ void mma_tt(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
    if constexpr (N == 64) wgmma_bf16_n64_tt(d, a, b, scale_d); else wgmma_bf16_n128_tt(d, a, b, scale_d);
}

template <int BN, int PASSES>
__global__ void __launch_bounds__(kWgThreads, 1)
conv_wgrad_tc_kernel(const __grid_constant__ CUtensorMap map_dy_hi, const __grid_constant__ CUtensorMap map_dy_lo,
                     const __grid_constant__ CUtensorMap map_x_hi, const __grid_constant__ CUtensorMap map_x_lo, const WgradParams p) {
    constexpr int STAGES = wg_num_stages(BN, PASSES), STAGE_BYTES = wg_stage_bytes(BN, PASSES);
    constexpr int NBOX = BN / 64;                                    // x boxes per plane and stage
    constexpr int X_OFF = (PASSES == 3 ? 2 : 1) * WG_BOX_BYTES;      // first x plane
    constexpr int X_PLANE = NBOX * WG_BOX_BYTES;
    constexpr int NR = BN / 2;
    static_assert(STAGES >= 4, "each consumer warpgroup holds two stages while the producer refills");
    static_assert(STAGES % 2 == 0, "one consumer warpgroup per stage (wg_num_stages)");
    static_assert(STAGES * STAGE_BYTES >= 64 * BN * 4, "the epilogue reduces the two fragments through the ring");
    static_assert(wg_smem_bytes(BN, PASSES) <= 227 * 1024, "conv_wgrad_tc_kernel: shared memory budget");

    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
    Ring ring{smem, bars, bars + STAGES, 0, 0};

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg = __shfl_sync(0xFFFFFFFFu, (int)threadIdx.x / 128, 0);
    const int tile = blockIdx.x % p.num_tiles, split = blockIdx.x / p.num_tiles;
    const int nt = tile % p.n_tiles, mt = (tile / p.n_tiles) % p.m_tiles, tap = tile / (p.n_tiles * p.m_tiles);
    const int kh = tap / p.k, kw = tap % p.k;
    const int pb0 = (int)((int64_t)split * p.pix_blocks / p.splits);
    const int nkb = (int)((int64_t)(split + 1) * p.pix_blocks / p.splits) - pb0;

    if (threadIdx.x == 0) {
        prefetch_tmap(&map_dy_hi); prefetch_tmap(&map_x_hi);
        if (PASSES == 3) { prefetch_tmap(&map_dy_lo); prefetch_tmap(&map_x_lo); }
        for (int s = 0; s < STAGES; ++s) { mbar_init(&ring.full[s], 1); mbar_init(&ring.empty[s], 4); }   // the 4 warps of one warpgroup
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (wg == 0) {
        setmaxnreg_dec<kWgProducerRegs>();
        if (warp == 0) {
            // ================================ TMA producer: K block kb of this split goes to stage kb % STAGES ================================
            for (int kb = 0; kb < nkb; ++kb) {
                const int pb = pb0 + kb;
                const int w0 = (pb % p.tiles_w) * p.TW, h0 = (pb / p.tiles_w % p.tiles_h) * p.TH, b0 = pb / (p.tiles_w * p.tiles_h) * p.TB;
                mbar_wait(&ring.empty[ring.stage], ring.phase ^ 1, p.err_flag, 1);
                H3D_SKEW(SKEW_PRODUCER, kb);
                if (elect_one()) {
                    uint8_t* st = ring.base + ring.stage * STAGE_BYTES;
                    uint64_t* fb = &ring.full[ring.stage];
                    mbar_expect_tx(fb, STAGE_BYTES);
                    tma_load_4d(&map_dy_hi, st, fb, mt * 64, w0, h0, b0);
                    if (PASSES == 3) tma_load_4d(&map_dy_lo, st + WG_BOX_BYTES, fb, mt * 64, w0, h0, b0);
#pragma unroll
                    for (int j = 0; j < NBOX; ++j) {
                        const int c0 = nt * BN + j * 64, xw = w0 + kw - p.pad, xh = h0 + kh - p.pad;
                        tma_load_4d(&map_x_hi, st + X_OFF + j * WG_BOX_BYTES, fb, c0, xw, xh, b0);
                        if (PASSES == 3) tma_load_4d(&map_x_lo, st + X_OFF + X_PLANE + j * WG_BOX_BYTES, fb, c0, xw, xh, b0);
                    }
                }
                __syncwarp();
                if (++ring.stage == STAGES) { ring.stage = 0; ring.phase ^= 1; }
            }
        }
    } else {
        setmaxnreg_inc<kWgConsumerRegs>();
        // ================================ wgmma: warpgroup cw takes the K blocks kb = cw, cw + 2, ... ================================
        const int cw = wg - 1;
        float racc[NR], acc[NR];
#pragma unroll
        for (int i = 0; i < NR; ++i) { racc[i] = 0.f; acc[i] = 0.f; }
        for (int kc = cw; kc < nkb; kc += 2 * p.chunk_kb) {   // chunks of chunk_kb of this warpgroup's K blocks
            const int kc_end = min(nkb, kc + 2 * p.chunk_kb);
            int pend = -1;
            for (int kb = kc; kb < kc_end; kb += 2) {
                const int stage = kb % STAGES;
                mbar_wait(&ring.full[stage], (uint32_t)(kb / STAGES) & 1u, p.err_flag, 3);
                H3D_SKEW(SKEW_CONSUMER, kb);
                const uint32_t sa = smem_u32(ring.base + stage * STAGE_BYTES);
                const uint64_t a_hi = desc_mn_sw128(sa, WG_BOX_BYTES), a_lo = desc_mn_sw128(sa + WG_BOX_BYTES, WG_BOX_BYTES);
                const uint64_t b_hi = desc_mn_sw128(sa + X_OFF, WG_BOX_BYTES), b_lo = desc_mn_sw128(sa + X_OFF + X_PLANE, WG_BOX_BYTES);
                fence_regs<NR>(acc);
                wgmma_fence();
#pragma unroll
                for (int j = 0; j < WG_ROWS / 16; ++j) {
                    const uint64_t koff = (uint64_t)j * (16 * 128 / 16);   // + 16 pixel rows (2048 bytes) per K step of 16
                    mma_tt<BN>(acc, a_hi + koff, b_hi + koff, (uint32_t)((kb > kc) | (j != 0)));
                    if (PASSES == 3) {
                        mma_tt<BN>(acc, a_hi + koff, b_lo + koff, 1u);
                        mma_tt<BN>(acc, a_lo + koff, b_hi + koff, 1u);
                    }
                }
                wgmma_commit();
                fence_regs<NR>(acc);
                H3D_SKEW(SKEW_COMMIT, kb);
                wgmma_wait<1>();
                if (pend >= 0 && lane == 0) mbar_arrive(&ring.empty[pend]);
                pend = stage;
            }
            wgmma_wait<0>();
            if (lane == 0) mbar_arrive(&ring.empty[pend]);
            fence_regs<NR>(acc);
#pragma unroll
            for (int i = 0; i < NR; ++i) racc[i] += acc[i];   // fold the chunk's tensor-core sum (round-to-nearest)
        }
        // ---- epilogue: fragment of warpgroup 2 through shared memory (the ring is idle: every stage has been consumed), added to
        // warpgroup 1's in a fixed order; thread t of both warpgroups holds the same fragment elements
        const int t = threadIdx.x & 127;
        float* red = reinterpret_cast<float*>(smem);
        H3D_SKEW(SKEW_EPILOGUE, 0);
        named_bar_sync(1, 256);
        if (cw == 1) {
#pragma unroll
            for (int i = 0; i < NR; ++i) red[i * 128 + t] = racc[i];
        }
        H3D_SKEW(SKEW_EPILOGUE, 1);
        named_bar_sync(1, 256);
        H3D_SKEW(SKEW_EPILOGUE, 2);
        if (cw == 0) {
            float* out = p.partial + ((int64_t)split * p.num_tiles + tile) * (64 * BN);
            const int m = 16 * (warp & 3) + (lane >> 2);
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {   // n8 block j: (m, n), (m, n + 1), (m + 8, n), (m + 8, n + 1)
                const int n = 8 * j + 2 * (lane & 3);
                out[n * 64 + m] = racc[4 * j] + red[(4 * j) * 128 + t];
                out[(n + 1) * 64 + m] = racc[4 * j + 1] + red[(4 * j + 1) * 128 + t];
                out[n * 64 + m + 8] = racc[4 * j + 2] + red[(4 * j + 2) * 128 + t];
                out[(n + 1) * 64 + m + 8] = racc[4 * j + 3] + red[(4 * j + 3) * 128 + t];
            }
        }
    }
}

// dW[tap][ci][co] (HWIO) = sum over the splits, in split order, of the CTA tiles' partial sums
__global__ void wgrad_reduce_kernel(const float* __restrict__ partial, float* __restrict__ dw, int kk, int Cin, int Cout, int m_tiles,
                                    int n_tiles, int BN, int splits) {
    const int num_tiles = kk * m_tiles * n_tiles;
    const int64_t total = (int64_t)kk * Cin * Cout;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int co = (int)(i % Cout), ci = (int)((i / Cout) % Cin), tap = (int)(i / ((int64_t)Cout * Cin));
        const int tile = (tap * m_tiles + co / 64) * n_tiles + ci / BN;
        const float* src = partial + (int64_t)tile * 64 * BN + (ci % BN) * 64 + co % 64;
        float s = 0.f;
        for (int sp = 0; sp < splits; ++sp) s += __ldg(src + (int64_t)sp * num_tiles * 64 * BN);
        dw[i] = s;
    }
}

// Device weight packing: HWIO fp32 -> 16-bit hi / lo planes with the rounding of the host packer (api.cu: pack_conv_weights).
//   forward:       [Cout_pad][k][k][Cin_pad],  element w[kh][kw][ci][co]
//   data gradient: [Cin_pad][k][k][Cout_pad],  element w[k-1-kh][k-1-kw][ci][co]
// bias_pad [rows] = the bias zero-padded to the row count (forward), or zeros (data gradient: the transposed convolution has no bias).
// w_scale (forward fp16 planes, else nullptr): the per-channel factors 2^-s of conv_w_shift_kernel; w / 2^-s is exact.
template <bool FP16>
__global__ void pack_conv_w_kernel(const float* __restrict__ w, const float* __restrict__ bias, uint16_t* __restrict__ hi,
                                   uint16_t* __restrict__ lo, float* __restrict__ bias_pad, const float* __restrict__ w_scale, int k,
                                   int Cin, int Cout, int Cin_pad, int Cout_pad, int dgrad) {
    const int kk = k * k;
    const int rows = dgrad ? Cin_pad : Cout_pad, cols = dgrad ? Cout_pad : Cin_pad;
    const int64_t total = (int64_t)rows * kk * cols;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % cols), tap = (int)((i / cols) % kk), r = (int)(i / ((int64_t)cols * kk));
        const int co = dgrad ? c : r, ci = dgrad ? r : c, src_tap = dgrad ? kk - 1 - tap : tap;
        float v = (co < Cout && ci < Cin) ? __ldg(w + ((int64_t)src_tap * Cin + ci) * Cout + co) : 0.f;
        if (w_scale) v = __fdiv_rn(v, w_scale[co]);
        uint16_t h;
        float hf;
        if (FP16) { h = __half_as_ushort(__float2half_rn(v)); hf = __half2float(__ushort_as_half(h)); }
        else { h = __bfloat16_as_ushort(__float2bfloat16_rn(v)); hf = __uint_as_float((uint32_t)h << 16); }
        hi[i] = h;
        if (lo) lo[i] = FP16 ? __half_as_ushort(__float2half_rn(v - hf)) : __bfloat16_as_ushort(__float2bfloat16_rn(v - hf));
        if (i < rows) bias_pad[i] = (!dgrad && bias && i < Cout) ? bias[i] : 0.f;
    }
}

// fp16 weight shifts (split_fmt.cuh): w_scale[co] = 2^-s(co) from max_k |w[k, co]|, 1 for the padding columns; one warp per column
__global__ void conv_w_shift_kernel(const float* __restrict__ w, float* __restrict__ w_scale, int K, int Cout, int Cout_pad) {
    const int co = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
    if (co >= Cout_pad) return;
    float mx = 0.f;
    if (co < Cout)
        for (int r = lane; r < K; r += 32) mx = fmaxf(mx, fabsf(__ldg(w + (int64_t)r * Cout + co)));
#pragma unroll
    for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xFFFFFFFFu, mx, o));
    if (lane == 0) w_scale[co] = ldexpf(1.f, -fp16_w_shift(mx));
}

// dy' = dy * act'(y) as bf16 split planes [B,H,W,Cout_pad] (input resolution; stride 2: dy' at the odd pixels, zeros elsewhere).
// Block b covers the pixels [b ppb, (b + 1) ppb), thread c channel c (blockDim.x = Cout_pad); db_part[b][c] = the block's column sum
// in pixel order.
template <bool LO>
__global__ void conv_grad_prep_kernel(const float* __restrict__ dy, const float* __restrict__ y, uint16_t* __restrict__ hi,
                                      uint16_t* __restrict__ lo, float* __restrict__ db_part, int B, int H, int W, int Cout, int stride,
                                      int leaky, int64_t ppb) {
    const int c = threadIdx.x, Cout_pad = blockDim.x;
    const int64_t P = (int64_t)B * H * W;
    const int64_t p0 = (int64_t)blockIdx.x * ppb, p1 = p0 + ppb < P ? p0 + ppb : P;
    const int Ho = H / stride, Wo = W / stride;
    float sum = 0.f;
    for (int64_t pix = p0; pix < p1; ++pix) {
        float v = 0.f;
        if (c < Cout) {
            int64_t src = pix;
            bool live = true;
            if (stride == 2) {
                const int w = (int)(pix % W), h = (int)((pix / W) % H), b = (int)(pix / ((int64_t)W * H));
                live = (w & 1) && (h & 1);
                src = ((int64_t)b * Ho + (h >> 1)) * Wo + (w >> 1);
            }
            if (live) {
                v = __ldg(dy + src * Cout + c);
                if (leaky && !(__ldg(y + src * Cout + c) >= 0.f)) v = v * kNegSlope;   // Maximum(x, 0.01 x): the 0.01 x branch
                sum += v;
            }
        }
        const uint16_t h = __bfloat16_as_ushort(__float2bfloat16_rn(v));
        hi[pix * Cout_pad + c] = h;
        if (LO) lo[pix * Cout_pad + c] = __bfloat16_as_ushort(__float2bfloat16_rn(v - __uint_as_float((uint32_t)h << 16)));
    }
    if (db_part) db_part[(int64_t)blockIdx.x * Cout_pad + c] = sum;
}

// db[c] = sum of the prep blocks' column sums: block c, fixed-order strided partials, then a fixed-order tree in shared memory
__global__ void bias_grad_reduce_kernel(const float* __restrict__ db_part, int nblk, int Cout_pad, float* __restrict__ db) {
    __shared__ float red[256];
    const int c = blockIdx.x, t = threadIdx.x;
    float s = 0.f;
    for (int b = t; b < nblk; b += 256) s += __ldg(db_part + (int64_t)b * Cout_pad + c);
    red[t] = s;
    __syncthreads();
    for (int h = 128; h > 0; h >>= 1) {
        if (t < h) red[t] += red[t + h];
        __syncthreads();
    }
    if (t == 0) db[c] = red[0];
}

struct WgradGeom { int TW, TH, TB, tiles_w, tiles_h, pix_blocks, BN, m_tiles, n_tiles, num_tiles, splits; };

// Pixel tile = one 64-pixel box (fewest boxes over the batch); BN = 128 where Cin_pad allows.  Split-K: the number of splits S (at most
// one per pixel block, S x tiles <= 8 x SMs) that fills the last wave of one-CTA-per-SM launches best; the smallest S on ties.
WgradGeom wgrad_geometry(int B, int H, int W, int k, int Cin_pad, int Cout_pad) {
    static const int cand[][3] = {{8, 8, 1}, {16, 4, 1}, {4, 16, 1}, {32, 2, 1}, {2, 32, 1}, {64, 1, 1}, {1, 64, 1}, {8, 4, 2},
                                  {4, 8, 2}, {4, 4, 4}, {4, 2, 8}, {2, 4, 8}, {2, 2, 16}, {1, 1, 64}};
    WgradGeom g{};
    int64_t best = -1;
    for (auto& c : cand) {
        const int64_t n = (int64_t)ceil_div(W, c[0]) * ceil_div(H, c[1]) * ceil_div(B, c[2]);
        if (best < 0 || n < best) { best = n; g.TW = c[0]; g.TH = c[1]; g.TB = c[2]; }
    }
    g.tiles_w = ceil_div(W, g.TW); g.tiles_h = ceil_div(H, g.TH);
    g.pix_blocks = (int)best;
    g.BN = Cin_pad % 128 == 0 ? 128 : 64;
    g.m_tiles = Cout_pad / 64; g.n_tiles = Cin_pad / g.BN;
    g.num_tiles = k * k * g.m_tiles * g.n_tiles;
    const int64_t sms = tc_num_sms(), T = g.num_tiles;
    auto eff = [&](int64_t S) { return (double)(S * T) / (double)(ceil_div64(S * T, sms) * sms); };
    g.splits = 1;
    for (int64_t S = 2; S <= g.pix_blocks && S * T <= 8 * sms; ++S)
        if (eff(S) > eff(g.splits) + 1e-6) g.splits = (int)S;
    return g;
}

template <int BN, int PASSES>
int launch_wgrad_inst(const CUtensorMap* maps, const WgradParams& p, cudaStream_t s) {
    constexpr int smem = wg_smem_bytes(BN, PASSES);
    static bool attr[64] = {};
    int dev = 0;
    H3D_CUDA(cudaGetDevice(&dev));
    if (!attr[dev % 64]) {
        H3D_CUDA(cudaFuncSetAttribute(conv_wgrad_tc_kernel<BN, PASSES>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        attr[dev % 64] = true;
    }
    conv_wgrad_tc_kernel<BN, PASSES><<<p.num_tiles * p.splits, kWgThreads, smem, s>>>(maps[0], maps[1], maps[2], maps[3], p);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

}  // namespace

int64_t conv_wgrad_partial_floats(int B, int H, int W, int k, int Cin_pad, int Cout_pad) {
    const WgradGeom g = wgrad_geometry(B, H, W, k, Cin_pad, Cout_pad);
    return (int64_t)g.splits * g.num_tiles * 64 * g.BN;
}

void conv_wgrad_geometry(int B, int H, int W, int k, int Cin_pad, int Cout_pad, int out[6]) {
    const WgradGeom g = wgrad_geometry(B, H, W, k, Cin_pad, Cout_pad);
    out[0] = g.TW; out[1] = g.TH; out[2] = g.TB; out[3] = g.BN; out[4] = g.num_tiles; out[5] = g.splits;
}

int launch_conv_wgrad(const WgradDesc& d, cudaStream_t s) {
    H3D_REQUIRE(d.passes == 1 || d.passes == 3, "conv_wgrad: 1 or 3 passes");
    H3D_REQUIRE(d.Cin_pad % 64 == 0 && d.Cout_pad % 64 == 0 && d.dy.hi && d.x.hi && (d.passes == 1 || (d.dy.lo && d.x.lo)),
                "conv_wgrad: bad operands");
    const WgradGeom g = wgrad_geometry(d.B, d.H, d.W, d.k, d.Cin_pad, d.Cout_pad);
    CUtensorMap maps[4];
    bool ok = encode_act_map(&maps[0], d.dy.hi, d.Cout_pad, d.Cout_pad, d.W, d.H, d.B, g.TW, g.TH, g.TB) &&
              encode_act_map(&maps[2], d.x.hi, d.Cin_pad, d.Cin_pad, d.W, d.H, d.B, g.TW, g.TH, g.TB);
    if (ok && d.passes == 3)
        ok = encode_act_map(&maps[1], d.dy.lo, d.Cout_pad, d.Cout_pad, d.W, d.H, d.B, g.TW, g.TH, g.TB) &&
             encode_act_map(&maps[3], d.x.lo, d.Cin_pad, d.Cin_pad, d.W, d.H, d.B, g.TW, g.TH, g.TB);
    if (!ok) return H3D_ECUDA;
    if (d.passes == 1) { maps[1] = maps[0]; maps[3] = maps[2]; }
    WgradParams p{};
    p.partial = d.partial;
    p.k = d.k; p.pad = d.k / 2; p.m_tiles = g.m_tiles; p.n_tiles = g.n_tiles; p.num_tiles = g.num_tiles; p.splits = g.splits;
    p.TW = g.TW; p.TH = g.TH; p.TB = g.TB; p.tiles_w = g.tiles_w; p.tiles_h = g.tiles_h; p.pix_blocks = g.pix_blocks;
    p.chunk_kb = d.passes == 3 ? 9 : 27;   // <= ~108 accumulating tensor-core steps per partial sum, as the forward
    p.err_flag = d.err_flag;
    int rc;
    if (g.BN == 128) rc = d.passes == 3 ? launch_wgrad_inst<128, 3>(maps, p, s) : launch_wgrad_inst<128, 1>(maps, p, s);
    else rc = d.passes == 3 ? launch_wgrad_inst<64, 3>(maps, p, s) : launch_wgrad_inst<64, 1>(maps, p, s);
    if (rc) return rc;
    const int64_t total = (int64_t)d.k * d.k * d.Cin * d.Cout;
    wgrad_reduce_kernel<<<(int)std::min<int64_t>(ceil_div64(total, 256), 132 * 32), 256, 0, s>>>(d.partial, d.dw, d.k * d.k, d.Cin, d.Cout,
                                                                                               g.m_tiles, g.n_tiles, g.BN, g.splits);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

int launch_pack_conv_w(const float* w_hwio, const float* bias, Split out, float* bias_pad, float* w_scale, int k, int Cin, int Cout,
                       int Cin_pad, int Cout_pad, bool dgrad, Half16 half, cudaStream_t s) {
    H3D_REQUIRE(!w_scale || (half == Half16::FP16 && !dgrad), "pack_conv_w: weight shifts belong to forward fp16 planes");
    const int64_t total = (int64_t)Cin_pad * Cout_pad * k * k;
    const int blocks = (int)std::min<int64_t>(ceil_div64(total, 256), 132 * 32);
    if (w_scale) {
        conv_w_shift_kernel<<<ceil_div(Cout_pad, 8), 256, 0, s>>>(w_hwio, w_scale, k * k * Cin, Cout, Cout_pad);
        H3D_CHECK_LAUNCH();
    }
    if (half == Half16::FP16)
        pack_conv_w_kernel<true><<<blocks, 256, 0, s>>>(w_hwio, bias, out.hi, out.lo, bias_pad, w_scale, k, Cin, Cout, Cin_pad, Cout_pad,
                                                        dgrad ? 1 : 0);
    else
        pack_conv_w_kernel<false><<<blocks, 256, 0, s>>>(w_hwio, bias, out.hi, out.lo, bias_pad, w_scale, k, Cin, Cout, Cin_pad, Cout_pad,
                                                         dgrad ? 1 : 0);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

int conv_grad_prep_blocks(int64_t pixels, int64_t* ppb) {
    const int64_t blocks = std::max<int64_t>(1, std::min<int64_t>(ceil_div64(pixels, 32), 4096));
    *ppb = ceil_div64(pixels, blocks);
    return (int)ceil_div64(pixels, *ppb);
}

int launch_conv_grad_prep(const float* dy, const float* y, Split out, float* db_part, int B, int H, int W, int Cout, int Cout_pad,
                          int stride, int leaky, cudaStream_t s) {
    H3D_REQUIRE(Cout_pad % 64 == 0 && Cout_pad <= 1024, "conv_grad_prep: Cout_pad must be a multiple of 64 and <= 1024");
    int64_t ppb = 0;
    const int nblk = conv_grad_prep_blocks((int64_t)B * H * W, &ppb);
    if (out.lo) conv_grad_prep_kernel<true><<<nblk, Cout_pad, 0, s>>>(dy, y, out.hi, out.lo, db_part, B, H, W, Cout, stride, leaky, ppb);
    else conv_grad_prep_kernel<false><<<nblk, Cout_pad, 0, s>>>(dy, y, out.hi, out.lo, db_part, B, H, W, Cout, stride, leaky, ppb);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

int launch_bias_grad_reduce(const float* db_part, int nblk, int Cout, int Cout_pad, float* db, cudaStream_t s) {
    bias_grad_reduce_kernel<<<Cout, 256, 0, s>>>(db_part, nblk, Cout_pad, db);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

}  // namespace h3d

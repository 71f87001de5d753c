// Philox4x64-10 and the fp32 uniform drawn from one of its words: the generator of the reader's augmentation (reader_aug.cu) and of
// the networks' dropout (dropout.cu).  Key and counter layouts are each caller's own (include/hand3d_b200.h).
#pragma once

#include <cstdint>

namespace h3d {

// Salmon, Moraes, Dror, Shaw, "Parallel random numbers: as easy as 1, 2, 3" (SC'11); the same function as numpy.random.Philox.
__device__ __forceinline__ void philox4x64_10(uint64_t c[4], uint64_t k0, uint64_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r) { k0 += 0x9E3779B97F4A7C15ull; k1 += 0xBB67AE8584CAA73Bull; }
        const uint64_t lo0 = 0xD2E7470EE14C6C93ull * c[0], hi0 = __umul64hi(0xD2E7470EE14C6C93ull, c[0]);
        const uint64_t lo1 = 0xCA5A826395121157ull * c[2], hi1 = __umul64hi(0xCA5A826395121157ull, c[2]);
        const uint64_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
        c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
    }
}

__device__ __forceinline__ float uniform01(uint64_t w) { return __fmul_rn((float)(w >> 40), 0x1p-24f); }     // exact

}  // namespace h3d

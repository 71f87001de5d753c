// EvalUtil (utils/general.py:522-611) on the device: a store of per-key-point distance lists that feeds append to without the host,
// and the measures get_measures() needs from each list, bit for bit with the reference's numpy.
//
// Feed: one CTA per key-point walks the batch's samples in order, computes each distance (keypoint_dist, common.cuh) and appends the
// visible ones at positions given by a block-wide prefix sum, so the lists grow in exactly the reference's per-sample append order.
// The last CTA to finish (a ticket in the header) advances the kept / dropped sample counters.
//
// Stats: one CTA per key-point.
//   - mean: numpy 2.x's pairwise_sum (umath/loops_utils.h.src) over the list, then / n in the list's dtype.  The recursion tree of
//     pairwise_sum is cut at a frontier of at most kFrontier subtrees: thread 0 enumerates them, every thread sums its subtrees with
//     the same recursion, and thread 0 combines the subtree sums along the top of the tree.  The summation order is numpy's.
//   - median: np.median's order statistics by radix select on the IEEE bit patterns (distances are +0 or above, so unsigned order is
//     value order), (a + b) / 2 in the list's dtype for even n, NaN if the list holds a NaN.
//   - counts: #{d <= threshold} with d promoted to float64, by binary search when the thresholds ascend (np.linspace), else by one
//     warp ballot per threshold.  Integer shared-memory atomics: the counts do not depend on their order.
#include "common.cuh"

namespace h3d {

namespace {

constexpr int kFeedThreads = 256;
constexpr int kStatsThreads = 512;
constexpr int kRadixBits = 11, kRadixBins = 1 << kRadixBits;
constexpr int kLeaf = 128;            // numpy's PW_BLOCKSIZE: a node of up to 128 values is summed with 8 accumulators
constexpr int kFrontier = 1024;
// Frontier: the largest nodes of length <= F = max(128, ceil(n / kFrontierSplit)).  A node longer than 128 splits into children of
// at least (L - 15) / 2 > 0.44 F values when L > F, so there are fewer than 2.3 * kFrontierSplit frontier nodes.
constexpr int kFrontierSplit = 384;
// pairwise_sum splits a node of L > 128 values into two of at least 64, so the depth for n <= 2^24 is at most 19: the node stack holds
// at most 2 * 19 + 1 entries and the value stack 20.
constexpr int kWalkStack = 40, kValueStack = 24;

static_assert(kRadixBins % kStatsThreads == 0, "radix bins per thread");

__device__ __forceinline__ uint32_t order_key(float x) { return isnan(x) ? 0xffffffffu : __float_as_uint(x); }
__device__ __forceinline__ uint64_t order_key(double x) { return isnan(x) ? ~0ull : (uint64_t)__double_as_longlong(x); }
__device__ __forceinline__ float key_value(uint32_t k) { return __uint_as_float(k); }
__device__ __forceinline__ double key_value(uint64_t k) { return __longlong_as_double((long long)k); }
__device__ __forceinline__ float rn_div(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double rn_div(double a, double b) { return __ddiv_rn(a, b); }

template <typename T> struct OrderKey;
template <> struct OrderKey<float> { using U = uint32_t; static constexpr int bits = 32; };
template <> struct OrderKey<double> { using U = uint64_t; static constexpr int bits = 64; };

// Exclusive prefix sum of one int per thread over the block; *total gets the block's sum.  Every thread must call it.
__device__ __forceinline__ int block_exclusive_scan(int v, int* s_warp, int* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(~0u, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
        int w = lane < nw ? s_warp[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(~0u, w, o);
            if (lane >= o) w += y;
        }
        if (lane < nw) s_warp[lane] = w;
    }
    __syncthreads();
    const int before = warp ? s_warp[warp - 1] : 0;
    *total = s_warp[nw - 1];
    __syncthreads();   // s_warp is free again when this returns
    return before + x - v;
}

template <typename T>
__global__ void __launch_bounds__(kFeedThreads) eval_feed_kernel(int64_t* __restrict__ hdr, T* __restrict__ data, int K, int N,
                                                                 const T* __restrict__ gt, const uint8_t* __restrict__ vis,
                                                                 const T* __restrict__ pred, int n, int D) {
    __shared__ int s_warp[32];
    __shared__ int64_t s_kept, s_cnt;
    const int k = blockIdx.x;
    if (threadIdx.x == 0) {       // read once, before this CTA takes its ticket below
        s_kept = hdr[H3D_EVAL_KEPT];
        s_cnt = hdr[H3D_EVAL_COUNT + k];
    }
    __syncthreads();
    const int64_t kept = s_kept;
    const int take = (int)min((int64_t)n, (int64_t)N - kept);   // samples past the store's capacity are dropped
    int64_t cnt = s_cnt;
    T* list = data + (int64_t)k * N;
    for (int base = 0; base < take; base += kFeedThreads) {
        const int r = base + threadIdx.x;
        const int64_t i = (int64_t)r * K + k;
        const bool v = r < take && vis[i] != 0;
        T d = T(0);
        if (v) d = keypoint_dist(gt + i * D, pred + i * D, D);
        int total;
        const int pos = block_exclusive_scan(v ? 1 : 0, s_warp, &total);
        if (v) list[cnt + pos] = d;
        cnt += total;
    }
    if (threadIdx.x == 0) {
        hdr[H3D_EVAL_COUNT + k] = cnt;
        __threadfence();
        // every CTA has read the sample counter before taking its ticket: the last one may advance it
        const unsigned long long t = atomicAdd(reinterpret_cast<unsigned long long*>(hdr + H3D_EVAL_TICKET), 1ull);
        if (t == (unsigned long long)(K - 1)) {
            hdr[H3D_EVAL_KEPT] = kept + take;
            hdr[H3D_EVAL_DROPPED] += n - take;
            hdr[H3D_EVAL_TICKET] = 0;
        }
    }
}

// numpy's pairwise_sum block: fewer than 8 values added in order from -0.0; else 8 accumulators over the blocks of 8 combined as
// ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the remainder in order.
template <typename T>
__device__ __forceinline__ T pairwise_leaf(const T* __restrict__ a, int n) {
    if (n < 8) {
        T r = T(-0.0);
        for (int i = 0; i < n; ++i) r = rn_add(r, a[i]);
        return r;
    }
    T r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = a[j];
    int i = 8;
    for (; i < n - (n % 8); i += 8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = rn_add(r[j], a[i + j]);
    }
    T res = rn_add(rn_add(rn_add(r[0], r[1]), rn_add(r[2], r[3])), rn_add(rn_add(r[4], r[5]), rn_add(r[6], r[7])));
    for (; i < n; ++i) res = rn_add(res, a[i]);
    return res;
}

// pairwise_sum's recursion over [off, off + len): a node of L > 128 values is the sum of its halves split at L/2 - (L/2) % 8, left plus
// right.  A node of at most F values is not split here; in left-to-right order the j-th such node is
//   kLeaves:    summed as pairwise_sum's block of a (F = 128, so every such node is a block);
//   kEnumerate: recorded as (s_off[j], s_len[j]) (while j < kFrontier) and valued 0; *count gets the number of nodes;
//   kCombine:   valued s_val[j].
// Explicit stacks: a node entry with len < 0 adds the two values on top of the value stack.
enum WalkMode { kLeaves, kEnumerate, kCombine };
template <WalkMode kMode, typename T>
__device__ __forceinline__ T pairwise_walk(const T* __restrict__ a, int off, int len, int F, int* s_off, int* s_len, const T* s_val,
                                           int* count) {
    int2 st[kWalkStack];
    T val[kValueStack];
    int sp = 0, vp = 0, j = 0;
    st[sp++] = make_int2(off, len);
    while (sp > 0) {
        const int2 e = st[--sp];
        const int o = e.x, l = e.y;
        if (l < 0) {
            val[vp - 2] = rn_add(val[vp - 2], val[vp - 1]);
            --vp;
        } else if (l <= F) {
            T v = T(0);
            if (kMode == kLeaves) {
                v = pairwise_leaf(a + o, l);
            } else if (kMode == kEnumerate) {
                if (j < kFrontier) { s_off[j] = o; s_len[j] = l; }
            } else {
                v = s_val[j];
            }
            ++j;
            val[vp++] = v;
        } else {
            int h = l / 2;
            h -= h % 8;
            st[sp++] = make_int2(o, -1);
            st[sp++] = make_int2(o + h, l - h);
            st[sp++] = make_int2(o, h);
        }
    }
    if (count) *count = j;
    return val[0];
}

// The key of rank `rank` (0-based, ascending) among the order keys of a[0, n), 11 bits per pass from the top.
template <typename T>
__device__ __forceinline__ typename OrderKey<T>::U radix_select(const T* __restrict__ a, int n, int rank, int* s_hist, int* s_warp, int* s_pick) {
    using U = typename OrderKey<T>::U;
    constexpr int per = kRadixBins / kStatsThreads;
    U prefix = 0, mask = 0;
    for (int hi = OrderKey<T>::bits; hi > 0; hi -= kRadixBits) {
        const int lo = max(hi - kRadixBits, 0);
        const U dmask = ((U)1 << (hi - lo)) - 1;
        for (int b = threadIdx.x; b < kRadixBins; b += kStatsThreads) s_hist[b] = 0;
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += kStatsThreads) {
            const U x = order_key(a[i]);
            if ((x & mask) == prefix) atomicAdd(&s_hist[(int)((x >> lo) & dmask)], 1);
        }
        __syncthreads();
        int c[per], sum = 0;
#pragma unroll
        for (int j = 0; j < per; ++j) {
            c[j] = s_hist[threadIdx.x * per + j];
            sum += c[j];
        }
        int total;
        int before = block_exclusive_scan(sum, s_warp, &total);
        if (before <= rank && rank < before + sum) {
#pragma unroll
            for (int j = 0; j < per; ++j) {
                if (rank >= before && rank < before + c[j]) {
                    s_pick[0] = threadIdx.x * per + j;
                    s_pick[1] = before;
                }
                before += c[j];
            }
        }
        __syncthreads();
        prefix |= (U)s_pick[0] << lo;
        mask |= dmask << lo;
        rank -= s_pick[1];
        __syncthreads();
    }
    return prefix;
}

template <typename T>
__global__ void __launch_bounds__(kStatsThreads, 1) eval_stats_kernel(const int64_t* __restrict__ hdr, const T* __restrict__ data, int N,
                                                                   const double* __restrict__ thr, int nthr, int64_t* __restrict__ out) {
    __shared__ int s_bins[H3D_EVAL_MAX_THRESHOLDS];
    __shared__ int s_hist[kRadixBins];
    __shared__ int s_off[kFrontier], s_len[kFrontier];
    __shared__ T s_val[kFrontier];
    __shared__ int s_warp[32], s_pick[2], s_m;
    const int k = blockIdx.x;
    const int n = (int)hdr[H3D_EVAL_COUNT + k];
    const T* a = data + (int64_t)k * N;
    int64_t* o = out + (int64_t)k * (H3D_EVAL_STAT_COUNTS + nthr);
    if (n == 0) {
        for (int i = threadIdx.x; i < H3D_EVAL_STAT_COUNTS + nthr; i += kStatsThreads) o[i] = 0;
        return;
    }

    // ---- counts[t] = #{d : float64(d) <= thr[t]}
    int unsorted = 0;
    for (int t = threadIdx.x; t < nthr; t += kStatsThreads) {
        s_bins[t] = 0;
        const double x = thr[t];
        if (isnan(x) || (t + 1 < nthr && !(x <= thr[t + 1]))) unsorted = 1;
    }
    unsorted = __syncthreads_or(unsorted);
    int has_nan = 0;
    if (!unsorted) {
        // a distance counts for every threshold from the first one it does not exceed: histogram of that index, then a prefix sum
        for (int i = threadIdx.x; i < n; i += kStatsThreads) {
            const T x = a[i];
            if (isnan(x)) { has_nan = 1; continue; }
            const double d = (double)x;
            int lo = 0, hi = nthr;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (d <= __ldg(thr + mid)) hi = mid;
                else lo = mid + 1;
            }
            if (lo < nthr) atomicAdd(&s_bins[lo], 1);
        }
        __syncthreads();
        int carry = 0;
        for (int base = 0; base < nthr; base += kStatsThreads) {
            const int t = base + threadIdx.x;
            const int v = t < nthr ? s_bins[t] : 0;
            int total;
            const int ex = block_exclusive_scan(v, s_warp, &total);
            if (t < nthr) o[H3D_EVAL_STAT_COUNTS + t] = carry + ex + v;
            carry += total;
        }
    } else {
        // thresholds in any order: a warp tests 32 distances against each threshold in turn
        const int lane = threadIdx.x & 31;
        for (int base = threadIdx.x & ~31; base < n; base += kStatsThreads) {
            const int i = base + lane;
            const bool in = i < n;
            const T x = in ? a[i] : T(0);
            if (in && isnan(x)) has_nan = 1;
            const double d = (double)x;
            for (int t = 0; t < nthr; ++t) {
                const unsigned m = __ballot_sync(~0u, in && d <= __ldg(thr + t));
                if (lane == 0 && m) atomicAdd(&s_bins[t], __popc(m));
            }
        }
        __syncthreads();
        for (int t = threadIdx.x; t < nthr; t += kStatsThreads) o[H3D_EVAL_STAT_COUNTS + t] = s_bins[t];
    }
    has_nan = __syncthreads_or(has_nan);

    // ---- mean: pairwise_sum in numpy's order, then / n
    const int F = max(kLeaf, (n + kFrontierSplit - 1) / kFrontierSplit);
    if (threadIdx.x == 0) {
        int m;
        pairwise_walk<kEnumerate>(a, 0, n, F, s_off, s_len, s_val, &m);
        s_m = min(m, kFrontier);
    }
    __syncthreads();
    for (int j = threadIdx.x; j < s_m; j += kStatsThreads)
        s_val[j] = pairwise_walk<kLeaves>(a, s_off[j], s_len[j], kLeaf, s_off, s_len, s_val, nullptr);
    __syncthreads();
    if (threadIdx.x == 0) {
        const T sum = pairwise_walk<kCombine>(a, 0, n, F, s_off, s_len, s_val, nullptr);
        o[H3D_EVAL_STAT_N] = n;
        o[H3D_EVAL_STAT_MEAN] = __double_as_longlong((double)rn_div(sum, (T)n));
    }

    // ---- median: the middle order statistic(s)
    T med;
    if (has_nan) {
        med = T(NAN);
    } else {
        const int r = (n - 1) / 2;
        const T lo = key_value(radix_select(a, n, r, s_hist, s_warp, s_pick));
        if (n & 1) {
            med = lo;
        } else {
            const T hi = key_value(radix_select(a, n, r + 1, s_hist, s_warp, s_pick));
            med = rn_div(rn_add(lo, hi), T(2));
        }
    }
    if (threadIdx.x == 0) o[H3D_EVAL_STAT_MEDIAN] = __double_as_longlong((double)med);
}

template <typename T>
int feed_typed(int64_t* hdr, T* data, int K, int N, const void* gt, const uint8_t* vis, const void* pred, int n, int D, cudaStream_t s) {
    eval_feed_kernel<T><<<K, kFeedThreads, 0, s>>>(hdr, data, K, N, static_cast<const T*>(gt), vis, static_cast<const T*>(pred), n, D);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

template <typename T>
int stats_typed(const int64_t* hdr, const T* data, int K, int N, const double* thr, int nthr, int64_t* out, cudaStream_t s) {
    eval_stats_kernel<T><<<K, kStatsThreads, 0, s>>>(hdr, data, N, thr, nthr, out);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

}  // namespace

int launch_eval_feed(void* store, int K, int N, int dtype, const void* gt, const uint8_t* vis, const void* pred, int n, int D,
                     cudaStream_t s) {
    int64_t* hdr = static_cast<int64_t*>(store);
    void* data = hdr + H3D_EVAL_HEADER_WORDS;
    if (dtype == H3D_EVAL_FLOAT64) return feed_typed(hdr, static_cast<double*>(data), K, N, gt, vis, pred, n, D, s);
    return feed_typed(hdr, static_cast<float*>(data), K, N, gt, vis, pred, n, D, s);
}

int launch_eval_stats(const void* store, int K, int N, int dtype, const double* thr, int nthr, int64_t* out, cudaStream_t s) {
    const int64_t* hdr = static_cast<const int64_t*>(store);
    const void* data = hdr + H3D_EVAL_HEADER_WORDS;
    if (dtype == H3D_EVAL_FLOAT64) return stats_typed(hdr, static_cast<const double*>(data), K, N, thr, nthr, out, s);
    return stats_typed(hdr, static_cast<const float*>(data), K, N, thr, nthr, out, s);
}

}  // namespace h3d

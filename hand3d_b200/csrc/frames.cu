// Camera frames in: run.py:57-59's scipy.misc.imresize(image_raw, (240, 320)) (Pillow's 8-bit BILINEAR resample) of uint8 RGB frames,
// bit for bit, optionally fused with run.py's normalisation float32(float64(u) / 255.0 - 0.5).
//
// Pillow's resample (libImaging/Resample.c): per axis a triangle filter of support max(in / out, 1), coefficients computed in double
// and normalised per output pixel, then converted to fixed point with 22 fractional bits (rounded half away from zero); every output
// value is (2^21 + sum of taps) >> 22 clipped to 0..255.  The horizontal pass runs first into a uint8 intermediate, then the vertical
// pass; an axis whose size does not change gets no pass.  The coefficients are built on the host once per (Hf, Wf, h, w) plan; this
// file is compiled with -ffp-contract=off so that the host never fuses a multiply-add into an FMA there.
//
// One kernel does both passes: a CTA owns one band of output rows of one image.  It streams the band's input rows (its rows plus the
// vertical filter's halo) from HBM through a double-buffered shared-memory stage (cp.async for the 16-byte words inside the row, byte
// loads at its unaligned ends), filters them horizontally into a uint8 chunk and adds each chunk's vertical contributions to int32
// accumulators of the band's output rows.  No intermediate leaves the SM.
//
// The kernel is instantiated per input pixel format (H3D_PIXEL_*; DESIGN.md section 4.18).  RGB and BGR stage the packed row; BGR only
// swaps the channels the horizontal pass writes.  The YUV formats stage each row's segments (NV12: the Y row and its interleaved UV row;
// I420: the Y row, its U row and its V row; YUYV: the packed row), each 16-byte aligned in its own slot, and convert them once per
// source pixel into an RGB chunk in shared memory (OpenCV's cvtColor BT.601 rule below), which the horizontal pass reads as the RGB
// instance reads its stage.  The plan pays for that chunk with fewer rows per stage.
#include <array>
#include <cstring>
#include <vector>

#include "common.cuh"

namespace h3d {

namespace {

constexpr int kFrameThreads = 512;
constexpr int kPrecisionBits = 22;                 // Pillow: 32 - 8 - 2
constexpr int kStageBudget = 28 * 1024;            // bytes per staging buffer (two of them)
constexpr int kAccBudget = 36 * 1024;              // bytes of int32 accumulators (the band's output rows)
constexpr int kMaxChunk = 8, kMaxBand = 16;

struct FrameArgs {
    const uint8_t* in;
    void* out;
    int Hf, Wf, h, w, normalize;
    int kxs, kys, band, chunk, row_stride, nbands;
    int acc_bytes, inter_bytes;
    const int32_t *xb, *kx, *yb, *ky;   // bounds (first tap, taps) and fixed-point coefficients per output column / row
    const float* lut;                   // [256] run.py's normalisation of each code
};
// The YUV formats' geometry: one frame's bytes, each segment's slot within a staged row, the converted RGB row's stride.  A kernel
// parameter of its own: growing FrameArgs changes the RGB instance's code (and made it 2-4 % slower on an H100).
struct YuvArgs {
    int64_t frame_bytes;
    int seg_off[3], rgb_stride;
};

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all_but_one() { asm volatile("cp.async.wait_group 1;\n" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;\n" ::: "memory"); }

// Byte j of input row r lands at buf[i * row_stride + (address of the row & 15) + j] (i = r - c0): the 16-byte words of the row keep
// their alignment in shared memory.  Words that lie wholly inside the row go through cp.async, the partial words at its ends byte by
// byte, so nothing outside the frames is read.
__device__ __forceinline__ void stage_rows(const FrameArgs& a, const uint8_t* img, int c0, int n, uint8_t* buf) {
    const int64_t rb = (int64_t)a.Wf * 3;
    const int words = a.row_stride >> 4;
    for (int k = threadIdx.x; k < n * words; k += kFrameThreads) {
        const int i = k / words, wd = k - i * words;
        const uintptr_t lo = (uintptr_t)(img + (int64_t)(c0 + i) * rb), hi = lo + (uintptr_t)rb;
        const uintptr_t g = (lo & ~(uintptr_t)15) + 16 * (uintptr_t)wd;
        uint8_t* d = buf + (int64_t)i * a.row_stride + 16 * wd;
        if (g >= lo && g + 16 <= hi) {
            cp_async16(d, (const void*)g);
        } else {
#pragma unroll
            for (int j = 0; j < 16; ++j)
                if (g + j >= lo && g + j < hi) d[j] = __ldg((const uint8_t*)(g + j));
        }
    }
}

__device__ __forceinline__ int clip8(int v) { return min(255, max(0, v >> kPrecisionBits)); }

constexpr bool is_yuv(int fmt) { return fmt == H3D_PIXEL_NV12 || fmt == H3D_PIXEL_I420 || fmt == H3D_PIXEL_YUYV; }
constexpr int n_segments(int fmt) { return fmt == H3D_PIXEL_I420 ? 3 : fmt == H3D_PIXEL_NV12 ? 2 : 1; }
constexpr int64_t frame_bytes_of(int fmt, int64_t H, int64_t W) {
    return fmt == H3D_PIXEL_NV12 || fmt == H3D_PIXEL_I420 ? H * W * 3 / 2 : fmt == H3D_PIXEL_YUYV ? H * W * 2 : H * W * 3;
}

// Segment s of input row r of a YUV frame (the planes and their layouts are in include/hand3d_b200.h) -> its first byte and length.
template <int FMT>
__device__ __forceinline__ const uint8_t* yuv_segment(const uint8_t* img, int Hf, int Wf, int s, int r, int& len) {
    const int64_t Y = (int64_t)Hf * Wf;
    if (FMT == H3D_PIXEL_YUYV) { len = 2 * Wf; return img + (int64_t)r * 2 * Wf; }
    if (s == 0) { len = Wf; return img + (int64_t)r * Wf; }
    if (FMT == H3D_PIXEL_NV12) { len = Wf; return img + Y + (int64_t)(r >> 1) * Wf; }
    len = Wf >> 1;                                                           // I420: U (s = 1) then V (s = 2)
    return img + Y + (s == 2 ? Y >> 2 : 0) + (int64_t)(r >> 1) * (Wf >> 1);
}

// stage_rows for the YUV formats: each segment of a row into its own slot, with the same alignment rule.
template <int FMT>
__device__ __forceinline__ void stage_yuv_rows(const FrameArgs& a, const YuvArgs& y, const uint8_t* img, int c0, int n, uint8_t* buf) {
#pragma unroll
    for (int sg = 0; sg < n_segments(FMT); ++sg) {
        const int words = (sg + 1 < n_segments(FMT) ? y.seg_off[sg + 1] - y.seg_off[sg] : a.row_stride - y.seg_off[sg]) >> 4;
        for (int k = threadIdx.x; k < n * words; k += kFrameThreads) {
            const int i = k / words, wd = k - i * words;
            int len;
            const uintptr_t lo = (uintptr_t)yuv_segment<FMT>(img, a.Hf, a.Wf, sg, c0 + i, len), hi = lo + (uintptr_t)len;
            const uintptr_t g = (lo & ~(uintptr_t)15) + 16 * (uintptr_t)wd;
            uint8_t* d = buf + (int64_t)i * a.row_stride + y.seg_off[sg] + 16 * wd;
            if (g >= lo && g + 16 <= hi) {
                cp_async16(d, (const void*)g);
            } else {
#pragma unroll
                for (int j = 0; j < 16; ++j)
                    if (g + j >= lo && g + j < hi) d[j] = __ldg((const uint8_t*)(g + j));
            }
        }
    }
}

// OpenCV's cvtColor COLOR_YUV2RGB_* (BT.601 limited range, 20-bit fixed point): one pixel from its luma and its block's chroma.
__device__ __forceinline__ void yuv_to_rgb(int Y, int U, int V, uint8_t* q) {
    const int c = max(Y - 16, 0) * 1220542 + (1 << 19), u = U - 128, v = V - 128;
    q[0] = (uint8_t)min(255, max(0, (c + 1673527 * v) >> 20));
    q[1] = (uint8_t)min(255, max(0, (c - 852492 * v - 409993 * u) >> 20));
    q[2] = (uint8_t)min(255, max(0, (c + 2116026 * u) >> 20));
}

// The luma of pixels 2p, 2p + 1 of a row and their shared chroma, read from the row's staged segments (st = the staged row).
template <int FMT>
__device__ __forceinline__ void yuv_pair(const FrameArgs& a, const YuvArgs& ya, const uint8_t* img, const uint8_t* st, int r, int p, int& y0,
                                         int& y1, int& u, int& v) {
    int len;
    const uint8_t* s0 = st + ya.seg_off[0] + ((uintptr_t)yuv_segment<FMT>(img, a.Hf, a.Wf, 0, r, len) & 15);
    if (FMT == H3D_PIXEL_YUYV) {
        y0 = s0[4 * p]; u = s0[4 * p + 1]; y1 = s0[4 * p + 2]; v = s0[4 * p + 3];
        return;
    }
    y0 = s0[2 * p]; y1 = s0[2 * p + 1];
    const uint8_t* s1 = st + ya.seg_off[1] + ((uintptr_t)yuv_segment<FMT>(img, a.Hf, a.Wf, 1, r, len) & 15);
    if (FMT == H3D_PIXEL_NV12) {
        u = s1[2 * p]; v = s1[2 * p + 1];
    } else {
        const uint8_t* s2 = st + ya.seg_off[2] + ((uintptr_t)yuv_segment<FMT>(img, a.Hf, a.Wf, 2, r, len) & 15);
        u = s1[p]; v = s2[p];
    }
}

// One CTA's work: output rows [band * a.band, +a.band) of output image b, read from the frame at img.  Shared by the batch kernel
// (one size and format per launch) and the rig kernel (a size per slot), force-inlined so that each keeps its own register allocation.
template <int FMT>
__device__ __forceinline__ void resize_band(const FrameArgs& a, const YuvArgs& ya, const uint8_t* img, int band, int64_t b) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int y0 = band * a.band, y1 = min(a.h, y0 + a.band), ny = y1 - y0;
    const int w3 = a.w * 3;
    int32_t* acc = reinterpret_cast<int32_t*>(smem);                     // [band][w3]
    uint8_t* inter = smem + a.acc_bytes;                                 // [chunk][w3]: the horizontal pass of the current chunk
    uint8_t* stage = inter + a.inter_bytes;                              // 2 x [chunk][row_stride]
    const int64_t stage_bytes = (int64_t)a.chunk * a.row_stride;
    uint8_t* rgb = stage + 2 * stage_bytes;                              // YUV formats: [chunk][rgb_stride], the converted chunk
    const int64_t rb = (int64_t)a.Wf * 3;
    const int r0 = a.yb[2 * y0], r1 = a.yb[2 * (y1 - 1)] + a.yb[2 * (y1 - 1) + 1];   // the band's input rows (bounds are monotone)
    const int nchunks = (r1 - r0 + a.chunk - 1) / a.chunk;

    for (int i = threadIdx.x; i < ny * w3; i += kFrameThreads) acc[i] = 1 << (kPrecisionBits - 1);
    if (is_yuv(FMT)) stage_yuv_rows<FMT>(a, ya, img, r0, min(a.chunk, r1 - r0), stage);
    else stage_rows(a, img, r0, min(a.chunk, r1 - r0), stage);
    cp_async_commit();
    for (int c = 0; c < nchunks; ++c) {
        const int c0 = r0 + c * a.chunk, n = min(a.chunk, r1 - c0);
        const uint8_t* cur = stage + (c & 1) * stage_bytes;
        if (c + 1 < nchunks) {        // the other buffer was last read before the barrier that ended the previous iteration
            if (is_yuv(FMT)) stage_yuv_rows<FMT>(a, ya, img, c0 + a.chunk, min(a.chunk, r1 - c0 - a.chunk), stage + ((c + 1) & 1) * stage_bytes);
            else stage_rows(a, img, c0 + a.chunk, min(a.chunk, r1 - c0 - a.chunk), stage + ((c + 1) & 1) * stage_bytes);
            cp_async_commit();
            cp_async_wait_all_but_one();
        } else {
            cp_async_wait_all();
        }
        __syncthreads();
        if (is_yuv(FMT)) {            // convert the chunk once per source pixel (two pixels, one chroma sample per thread)
            const int np = a.Wf >> 1;
            for (int i = threadIdx.x; i < n * np; i += kFrameThreads) {
                const int r = i / np, p = i - r * np;
                int y0p, y1p, u, v;
                yuv_pair<FMT>(a, ya, img, cur + (int64_t)r * a.row_stride, c0 + r, p, y0p, y1p, u, v);
                uint8_t* q = rgb + (int64_t)r * ya.rgb_stride + 6 * p;
                yuv_to_rgb(y0p, u, v, q);
                yuv_to_rgb(y1p, u, v, q + 3);
            }
            __syncthreads();
        }
        // horizontal pass: n input rows x w output columns, three channels per thread (one coefficient load per tap)
        for (int i = threadIdx.x; i < n * a.w; i += kFrameThreads) {
            const int r = i / a.w, x = i - r * a.w;
            const int off = is_yuv(FMT) ? 0 : (int)((uintptr_t)(img + (int64_t)(c0 + r) * rb) & 15);
            const int xmin = __ldg(a.xb + 2 * x), nx = __ldg(a.xb + 2 * x + 1);
            const int32_t* k = a.kx + (int64_t)x * a.kxs;
            const uint8_t* p = is_yuv(FMT) ? rgb + (int64_t)r * ya.rgb_stride + xmin * 3 : cur + (int64_t)r * a.row_stride + off + xmin * 3;
            int s0 = 1 << (kPrecisionBits - 1), s1 = s0, s2 = s0;
            for (int t = 0; t < nx; ++t) {
                const int kt = __ldg(k + t);
                s0 += p[3 * t] * kt;
                s1 += p[3 * t + 1] * kt;
                s2 += p[3 * t + 2] * kt;
            }
            if (FMT == H3D_PIXEL_BGR) { const int t = s0; s0 = s2; s2 = t; }
            uint8_t* q = inter + r * w3 + 3 * x;
            q[0] = (uint8_t)clip8(s0); q[1] = (uint8_t)clip8(s1); q[2] = (uint8_t)clip8(s2);
        }
        __syncthreads();
        // vertical pass: the chunk's contributions to every output row of the band whose taps reach into it
        for (int y = y0; y < y1; ++y) {
            const int ymin = __ldg(a.yb + 2 * y), yend = ymin + __ldg(a.yb + 2 * y + 1);
            const int lo = max(c0, ymin), hi = min(c0 + n, yend);
            if (lo >= hi) continue;
            const int32_t* k = a.ky + (int64_t)y * a.kys + (lo - ymin);
            for (int xc = threadIdx.x; xc < w3; xc += kFrameThreads) {
                int s = 0;
                for (int r = lo; r < hi; ++r) s += inter[(r - c0) * w3 + xc] * __ldg(k + (r - lo));
                acc[(y - y0) * w3 + xc] += s;
            }
        }
        __syncthreads();
    }
    const int64_t o = (b * a.h + y0) * (int64_t)w3;   // the band's output rows are contiguous
    if (a.normalize) {
        float* out = static_cast<float*>(a.out) + o;
        for (int i = threadIdx.x; i < ny * w3; i += kFrameThreads) out[i] = __ldg(a.lut + clip8(acc[i]));
    } else {
        uint8_t* out = static_cast<uint8_t*>(a.out) + o;
        for (int i = threadIdx.x; i < ny * w3; i += kFrameThreads) out[i] = (uint8_t)clip8(acc[i]);
    }
}

template <int FMT>
__global__ void __launch_bounds__(kFrameThreads, 2) resize_frames_kernel(FrameArgs a, YuvArgs ya) {
    const int band = blockIdx.x % a.nbands;
    const int64_t b = blockIdx.x / a.nbands;
    const uint8_t* img = is_yuv(FMT) ? a.in + b * ya.frame_bytes : a.in + b * a.Hf * ((int64_t)a.Wf * 3);
    resize_band<FMT>(a, ya, img, band, b);
}

// A camera rig (DESIGN.md section 4.19): the slots of one format, each with its own size, in one launch.  The plan's table (in device
// memory) holds each slot's geometry and coefficient offsets; the frame pointers are kernel parameters, so the plan serves any buffers.
struct RigArgs {
    const int32_t* table;    // include/hand3d_b200.h: B slot records, the order [B], the launch records
    const int32_t* coef;     // the normalisation table, then the coefficient tables of each distinct size
    void* out;
    int B, h, w, normalize, first, nslots;    // first: this launch's first position in the order
    const uint8_t* in[H3D_FRAME_RIG_MAX_SLOTS];
};

// The slot's arguments are read once into shared memory, where the band reads them as the batch kernel reads its parameters: held
// in registers, they would not fit the 64 that two CTAs per SM leave.
template <int FMT>
__global__ void __launch_bounds__(kFrameThreads, 2) resize_frames_rig_kernel(const __grid_constant__ RigArgs r) {
    __shared__ FrameArgs a;
    __shared__ YuvArgs ya;
    __shared__ int slot, band;
    if (threadIdx.x == 0) {
        const int32_t* order = r.table + (int64_t)r.B * H3D_FRAME_RIG_SLOT_WORDS + r.first;
        int i = 0;           // the launch's slots cover consecutive CTA ranges in order: the last one starting at or before this CTA
        while (i + 1 < r.nslots && r.table[order[i + 1] * H3D_FRAME_RIG_SLOT_WORDS + H3D_RIG_CTA0] <= (int)blockIdx.x) ++i;
        const int b = order[i];
        const int32_t* e = r.table + b * H3D_FRAME_RIG_SLOT_WORDS;
        a.in = r.in[b]; a.out = r.out; a.Hf = e[H3D_RIG_H]; a.Wf = e[H3D_RIG_W]; a.h = r.h; a.w = r.w; a.normalize = r.normalize;
        a.kxs = e[H3D_RIG_KXS]; a.kys = e[H3D_RIG_KYS]; a.band = e[H3D_RIG_BAND]; a.chunk = e[H3D_RIG_CHUNK];
        a.row_stride = e[H3D_RIG_ROW_STRIDE]; a.nbands = e[H3D_RIG_NBANDS];
        a.acc_bytes = e[H3D_RIG_ACC_BYTES]; a.inter_bytes = e[H3D_RIG_INTER_BYTES];
        a.xb = r.coef + e[H3D_RIG_XB]; a.kx = r.coef + e[H3D_RIG_KX]; a.yb = r.coef + e[H3D_RIG_YB]; a.ky = r.coef + e[H3D_RIG_KY];
        a.lut = reinterpret_cast<const float*>(r.coef);
        ya.frame_bytes = 0;
        for (int k = 0; k < 3; ++k) ya.seg_off[k] = e[H3D_RIG_SEG_OFF + k];
        ya.rgb_stride = e[H3D_RIG_RGB_STRIDE];
        slot = b;
        band = (int)blockIdx.x - e[H3D_RIG_CTA0];
    }
    __syncthreads();
    resize_band<FMT>(a, ya, a.in, band, slot);
}

// Full-size conversion of any format into packed RGB: one thread per chroma block (2x2 for NV12 and I420, 2x1 for YUYV; one pixel for
// RGB and BGR), consecutive threads on consecutive blocks of a row pair.
template <int FMT>
__global__ void __launch_bounds__(256) convert_frames_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int H, int W,
                                                             int64_t blocks) {
    constexpr int BH = FMT == H3D_PIXEL_NV12 || FMT == H3D_PIXEL_I420 ? 2 : 1, BW = is_yuv(FMT) ? 2 : 1;
    const int bw = W / BW, bh = H / BH;
    const int64_t per_image = (int64_t)bw * bh;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < blocks; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t b = i / per_image;
        const int64_t j = i - b * per_image;
        const int by = (int)(j / bw), bx = (int)(j - (int64_t)by * bw);
        const uint8_t* img = in + b * frame_bytes_of(FMT, H, W);
        uint8_t* q = out + ((b * H + (int64_t)by * BH) * W + (int64_t)bx * BW) * 3;
        if (FMT == H3D_PIXEL_RGB || FMT == H3D_PIXEL_BGR) {
            const uint8_t* p = img + ((int64_t)by * W + bx) * 3;
            const uint8_t c0 = p[0], c1 = p[1], c2 = p[2];
            q[0] = FMT == H3D_PIXEL_BGR ? c2 : c0; q[1] = c1; q[2] = FMT == H3D_PIXEL_BGR ? c0 : c2;
        } else if (FMT == H3D_PIXEL_YUYV) {
            const uint8_t* p = img + ((int64_t)by * W + 2 * bx) * 2;
            const int y0 = p[0], u = p[1], y1 = p[2], v = p[3];
            yuv_to_rgb(y0, u, v, q);
            yuv_to_rgb(y1, u, v, q + 3);
        } else {
            const int64_t Y = (int64_t)H * W;
            const uint8_t* yp = img + (int64_t)2 * by * W + 2 * bx;
            int u, v;
            if (FMT == H3D_PIXEL_NV12) {
                const uint8_t* c = img + Y + (int64_t)by * W + 2 * bx;
                u = c[0]; v = c[1];
            } else {
                const int64_t ci = (int64_t)by * (W / 2) + bx;
                u = img[Y + ci]; v = img[Y + Y / 4 + ci];
            }
            yuv_to_rgb(yp[0], u, v, q);
            yuv_to_rgb(yp[1], u, v, q + 3);
            yuv_to_rgb(yp[W], u, v, q + (int64_t)W * 3);
            yuv_to_rgb(yp[W + 1], u, v, q + (int64_t)W * 3 + 3);
        }
    }
}

// Pillow's precompute_coeffs + normalize_coeffs_8bpc for the bilinear filter (support 1) over a whole axis.  An axis that keeps its
// size gets one tap of weight 1 per pixel (Pillow does not resample it: a copy).  bounds[2i] = first input pixel, bounds[2i+1] = taps.
int pil_bilinear_coeffs(int in, int out, std::vector<int32_t>& bounds, std::vector<int32_t>& kk) {
    bounds.assign(2 * (size_t)out, 0);
    if (in == out) {
        kk.assign((size_t)out, 1 << kPrecisionBits);
        for (int i = 0; i < out; ++i) { bounds[2 * i] = i; bounds[2 * i + 1] = 1; }
        return 1;
    }
    const double scale = (double)in / (double)out;
    const double filterscale = scale < 1.0 ? 1.0 : scale;
    const double support = 1.0 * filterscale;
    const int ksize = (int)std::ceil(support) * 2 + 1;
    const double ss = 1.0 / filterscale;
    kk.assign((size_t)out * ksize, 0);
    std::vector<double> k((size_t)ksize);
    for (int xx = 0; xx < out; ++xx) {
        const double center = (xx + 0.5) * scale;
        int xmin = (int)(center - support + 0.5);
        if (xmin < 0) xmin = 0;
        int xmax = (int)(center + support + 0.5);
        if (xmax > in) xmax = in;
        xmax -= xmin;
        double ww = 0.0;
        for (int x = 0; x < xmax; ++x) {
            double t = (x + xmin - center + 0.5) * ss;
            if (t < 0.0) t = -t;
            const double w = t < 1.0 ? 1.0 - t : 0.0;
            k[x] = w;
            ww += w;
        }
        for (int x = 0; x < xmax; ++x)
            if (ww != 0.0) k[x] /= ww;
        for (int x = 0; x < xmax; ++x)
            kk[(size_t)xx * ksize + x] = k[x] < 0 ? (int32_t)(-0.5 + k[x] * (1 << kPrecisionBits)) : (int32_t)(0.5 + k[x] * (1 << kPrecisionBits));
        bounds[2 * xx] = xmin;
        bounds[2 * xx + 1] = xmax;
    }
    return ksize;
}

}  // namespace

struct FramePlan {
    int fmt = H3D_PIXEL_RGB, Hf = 0, Wf = 0, h = 0, w = 0;
    int kxs = 0, kys = 0, band = 0, chunk = 0, row_stride = 0, nbands = 0, acc_bytes = 0, inter_bytes = 0, smem = 0;
    int seg_off[3] = {0, 0, 0}, rgb_stride = 0;
    std::vector<int32_t> host;      // the source of the asynchronous upload, kept for the plan's lifetime
    int32_t* dev = nullptr;         // [xb | kx | yb | ky | lut]
    const int32_t *xb = nullptr, *kx = nullptr, *yb = nullptr, *ky = nullptr;
    const float* lut = nullptr;
};

namespace {

const void* resize_kernel_of(int fmt) {
    switch (fmt) {
        case H3D_PIXEL_BGR: return (const void*)resize_frames_kernel<H3D_PIXEL_BGR>;
        case H3D_PIXEL_NV12: return (const void*)resize_frames_kernel<H3D_PIXEL_NV12>;
        case H3D_PIXEL_I420: return (const void*)resize_frames_kernel<H3D_PIXEL_I420>;
        case H3D_PIXEL_YUYV: return (const void*)resize_frames_kernel<H3D_PIXEL_YUYV>;
        default: return (const void*)resize_frames_kernel<H3D_PIXEL_RGB>;
    }
}

// The launch geometry of a plan of p.fmt, p.Hf x p.Wf -> p.h x p.w (p.kxs and p.kys set): shared by single-size plans and rig slots.
void frame_geometry(FramePlan& p) {
    const int w3 = 3 * p.w;
    if (is_yuv(p.fmt)) {
        // a staged row is one 16-byte aligned slot per segment; the converted chunk takes its share of both stage buffers' budget
        const int n = p.fmt == H3D_PIXEL_I420 ? 3 : p.fmt == H3D_PIXEL_NV12 ? 2 : 1;
        const int len[3] = {p.fmt == H3D_PIXEL_YUYV ? 2 * p.Wf : p.Wf, p.fmt == H3D_PIXEL_NV12 ? p.Wf : p.Wf / 2, p.Wf / 2};
        for (int i = 0; i < n; ++i) {
            p.seg_off[i] = p.row_stride;
            p.row_stride += (int)align_up((int64_t)len[i] + 15, 16);
        }
        p.rgb_stride = (int)align_up((int64_t)p.Wf * 3, 16);
        p.chunk = std::max(1, std::min(kMaxChunk, 2 * kStageBudget / (2 * p.row_stride + p.rgb_stride)));
    } else {
        p.row_stride = (int)align_up((int64_t)p.Wf * 3 + 15, 16);
        p.chunk = std::max(1, std::min(kMaxChunk, kStageBudget / p.row_stride));
    }
    p.band = std::max(1, std::min({kMaxBand, p.h, kAccBudget / (w3 * 4)}));
    p.nbands = ceil_div(p.h, p.band);
    p.acc_bytes = (int)align_up((int64_t)p.band * w3 * 4, 16);
    p.inter_bytes = (int)align_up((int64_t)p.chunk * w3, 16);
    p.smem = p.acc_bytes + p.inter_bytes + 2 * p.chunk * p.row_stride + p.chunk * p.rgb_stride;
}

}  // namespace

FramePlan* frame_plan_create(int fmt, int Hf, int Wf, int h, int w, cudaStream_t s) {
    auto* p = new FramePlan();
    p->fmt = fmt; p->Hf = Hf; p->Wf = Wf; p->h = h; p->w = w;
    std::vector<int32_t> xb, kx, yb, ky;
    p->kxs = pil_bilinear_coeffs(Wf, w, xb, kx);
    p->kys = pil_bilinear_coeffs(Hf, h, yb, ky);
    frame_geometry(*p);
    auto& v = p->host;
    const size_t oxb = 0, okx = oxb + xb.size(), oyb = okx + kx.size(), oky = oyb + yb.size(), olut = oky + ky.size();
    v.resize(olut + 256);
    std::copy(xb.begin(), xb.end(), v.begin() + oxb);
    std::copy(kx.begin(), kx.end(), v.begin() + okx);
    std::copy(yb.begin(), yb.end(), v.begin() + oyb);
    std::copy(ky.begin(), ky.end(), v.begin() + oky);
    for (int u = 0; u < 256; ++u) {    // run.py:59: image_raw.astype('float') / 255.0 - 0.5 in double, then the float32 input
        const float f = (float)((double)u / 255.0 - 0.5);
        memcpy(&v[olut + u], &f, 4);
    }
    // the attribute is per kernel, not per plan: only ever raise it, or a plan with less shared memory would break the earlier ones
    cudaFuncAttributes fa;
    const void* kern = resize_kernel_of(fmt);
    cudaError_t e = cudaFuncGetAttributes(&fa, kern);
    if (e == cudaSuccess && fa.maxDynamicSharedSizeBytes < p->smem)
        e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, p->smem);
    if (e == cudaSuccess) e = cudaMalloc(&p->dev, v.size() * 4);
    if (e == cudaSuccess) e = cudaMemcpyAsync(p->dev, v.data(), v.size() * 4, cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) {
        cuda_fail(e, "frame_plan_create", __FILE__, __LINE__);
        frame_plan_destroy(p);
        return nullptr;
    }
    p->xb = p->dev + oxb; p->kx = p->dev + okx; p->yb = p->dev + oyb; p->ky = p->dev + oky;
    p->lut = reinterpret_cast<const float*>(p->dev + olut);
    return p;
}

void frame_plan_destroy(FramePlan* p) {
    if (!p) return;
    if (p->dev) cudaFree(p->dev);
    delete p;
}

int launch_resize_frames(const FramePlan* p, const uint8_t* frames, int B, int normalize, void* out, cudaStream_t s) {
    const int64_t grid = (int64_t)B * p->nbands;
    if (grid >= (1ll << 31)) {
        set_error("h3d_resize_frames: B = %d frames of %dx%d is too many for one launch", B, p->Hf, p->Wf);
        return H3D_EINVAL;
    }
    FrameArgs a;
    a.in = frames; a.out = out; a.Hf = p->Hf; a.Wf = p->Wf; a.h = p->h; a.w = p->w; a.normalize = normalize;
    a.kxs = p->kxs; a.kys = p->kys; a.band = p->band; a.chunk = p->chunk; a.row_stride = p->row_stride; a.nbands = p->nbands;
    a.acc_bytes = p->acc_bytes; a.inter_bytes = p->inter_bytes;
    YuvArgs y;
    for (int i = 0; i < 3; ++i) y.seg_off[i] = p->seg_off[i];
    y.rgb_stride = p->rgb_stride;
    y.frame_bytes = frame_bytes_of(p->fmt, p->Hf, p->Wf);
    a.xb = p->xb; a.kx = p->kx; a.yb = p->yb; a.ky = p->ky; a.lut = p->lut;
    switch (p->fmt) {
        case H3D_PIXEL_BGR: resize_frames_kernel<H3D_PIXEL_BGR><<<(unsigned)grid, kFrameThreads, p->smem, s>>>(a, y); break;
        case H3D_PIXEL_NV12: resize_frames_kernel<H3D_PIXEL_NV12><<<(unsigned)grid, kFrameThreads, p->smem, s>>>(a, y); break;
        case H3D_PIXEL_I420: resize_frames_kernel<H3D_PIXEL_I420><<<(unsigned)grid, kFrameThreads, p->smem, s>>>(a, y); break;
        case H3D_PIXEL_YUYV: resize_frames_kernel<H3D_PIXEL_YUYV><<<(unsigned)grid, kFrameThreads, p->smem, s>>>(a, y); break;
        default: resize_frames_kernel<H3D_PIXEL_RGB><<<(unsigned)grid, kFrameThreads, p->smem, s>>>(a, y); break;
    }
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

int launch_convert_frames(const uint8_t* frames, int fmt, int B, int H, int W, uint8_t* out, cudaStream_t s) {
    const int per_block = fmt == H3D_PIXEL_NV12 || fmt == H3D_PIXEL_I420 ? 4 : fmt == H3D_PIXEL_YUYV ? 2 : 1;
    const int64_t blocks = (int64_t)B * H * W / per_block;
    const int64_t grid = std::min<int64_t>(ceil_div64(blocks, 256), 1 << 20);   // grid-stride beyond
    switch (fmt) {
        case H3D_PIXEL_BGR: convert_frames_kernel<H3D_PIXEL_BGR><<<(unsigned)grid, 256, 0, s>>>(frames, out, H, W, blocks); break;
        case H3D_PIXEL_NV12: convert_frames_kernel<H3D_PIXEL_NV12><<<(unsigned)grid, 256, 0, s>>>(frames, out, H, W, blocks); break;
        case H3D_PIXEL_I420: convert_frames_kernel<H3D_PIXEL_I420><<<(unsigned)grid, 256, 0, s>>>(frames, out, H, W, blocks); break;
        case H3D_PIXEL_YUYV: convert_frames_kernel<H3D_PIXEL_YUYV><<<(unsigned)grid, 256, 0, s>>>(frames, out, H, W, blocks); break;
        default: convert_frames_kernel<H3D_PIXEL_RGB><<<(unsigned)grid, 256, 0, s>>>(frames, out, H, W, blocks); break;
    }
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

// ---- camera rigs (DESIGN.md section 4.19)

struct FrameRigPlan {
    int B = 0, h = 0, w = 0;
    int launch[H3D_PIXEL_YUYV + 1][H3D_FRAME_RIG_LAUNCH_WORDS] = {};
    std::vector<int32_t> host;      // [table | coef], the source of the asynchronous upload, kept for the plan's lifetime
    int32_t* dev = nullptr;
    const int32_t *table = nullptr, *coef = nullptr;
};

namespace {

const void* rig_kernel_of(int fmt) {
    switch (fmt) {
        case H3D_PIXEL_BGR: return (const void*)resize_frames_rig_kernel<H3D_PIXEL_BGR>;
        case H3D_PIXEL_NV12: return (const void*)resize_frames_rig_kernel<H3D_PIXEL_NV12>;
        case H3D_PIXEL_I420: return (const void*)resize_frames_rig_kernel<H3D_PIXEL_I420>;
        case H3D_PIXEL_YUYV: return (const void*)resize_frames_rig_kernel<H3D_PIXEL_YUYV>;
        default: return (const void*)resize_frames_rig_kernel<H3D_PIXEL_RGB>;
    }
}

}  // namespace

// include/hand3d_b200.h's rig table and coefficient buffer; the caller has checked the formats and sizes.  Each distinct (H, W) gets
// its coefficients once, from the same host code (and the same -ffp-contract=off) as a single-size plan.
void frame_rig_layout(int B, const int* fmt, const int* hw, int h, int w, std::vector<int32_t>& table, std::vector<int32_t>& coef) {
    constexpr int SW = H3D_FRAME_RIG_SLOT_WORDS, LW = H3D_FRAME_RIG_LAUNCH_WORDS;
    table.assign((size_t)B * SW + B + (H3D_PIXEL_YUYV + 1) * LW, 0);
    coef.assign(256, 0);
    for (int u = 0; u < 256; ++u) {
        const float f = (float)((double)u / 255.0 - 0.5);
        memcpy(&coef[u], &f, 4);
    }
    std::vector<std::array<int, 8>> sizes;   // H, W, then the offsets of xb, kx, yb, ky and kxs, kys
    for (int b = 0; b < B; ++b) {
        const int H = hw[2 * b], W = hw[2 * b + 1];
        int si = 0;
        while (si < (int)sizes.size() && (sizes[si][0] != H || sizes[si][1] != W)) ++si;
        if (si == (int)sizes.size()) {
            std::vector<int32_t> xb, kx, yb, ky;
            std::array<int, 8> z{H, W, 0, 0, 0, 0, 0, 0};
            z[6] = pil_bilinear_coeffs(W, w, xb, kx);
            z[7] = pil_bilinear_coeffs(H, h, yb, ky);
            for (int t = 0; t < 4; ++t) {
                const std::vector<int32_t>& v = t == 0 ? xb : t == 1 ? kx : t == 2 ? yb : ky;
                z[2 + t] = (int)coef.size();
                coef.insert(coef.end(), v.begin(), v.end());
            }
            sizes.push_back(z);
        }
        FramePlan g;
        g.fmt = fmt[b]; g.Hf = H; g.Wf = W; g.h = h; g.w = w; g.kxs = sizes[si][6]; g.kys = sizes[si][7];
        frame_geometry(g);
        int32_t* e = &table[(size_t)b * SW];
        e[H3D_RIG_FORMAT] = g.fmt; e[H3D_RIG_H] = H; e[H3D_RIG_W] = W; e[H3D_RIG_KXS] = g.kxs; e[H3D_RIG_KYS] = g.kys;
        e[H3D_RIG_BAND] = g.band; e[H3D_RIG_CHUNK] = g.chunk; e[H3D_RIG_ROW_STRIDE] = g.row_stride; e[H3D_RIG_NBANDS] = g.nbands;
        e[H3D_RIG_ACC_BYTES] = g.acc_bytes; e[H3D_RIG_INTER_BYTES] = g.inter_bytes; e[H3D_RIG_SMEM] = g.smem;
        for (int k = 0; k < 3; ++k) e[H3D_RIG_SEG_OFF + k] = g.seg_off[k];
        e[H3D_RIG_RGB_STRIDE] = g.rgb_stride;
        for (int t = 0; t < 4; ++t) e[H3D_RIG_XB + t] = sizes[si][2 + t];
        e[H3D_RIG_SIZE] = si;
    }
    int32_t* order = &table[(size_t)B * SW];
    int32_t* launch = order + B;
    int pos = 0;
    for (int f = 0; f <= H3D_PIXEL_YUYV; ++f) {
        int32_t* l = launch + f * LW;
        l[H3D_RIG_LAUNCH_FIRST] = pos;
        for (int b = 0; b < B; ++b) {
            int32_t* e = &table[(size_t)b * SW];
            if (e[H3D_RIG_FORMAT] != f) continue;
            order[pos++] = b;
            e[H3D_RIG_CTA0] = l[H3D_RIG_LAUNCH_CTAS];
            l[H3D_RIG_LAUNCH_SLOTS] += 1;
            l[H3D_RIG_LAUNCH_CTAS] += e[H3D_RIG_NBANDS];
            l[H3D_RIG_LAUNCH_SMEM] = std::max(l[H3D_RIG_LAUNCH_SMEM], e[H3D_RIG_SMEM]);
        }
    }
}

FrameRigPlan* frame_rig_plan_create(int B, const int* fmt, const int* hw, int h, int w, cudaStream_t s) {
    auto* p = new FrameRigPlan();
    p->B = B; p->h = h; p->w = w;
    std::vector<int32_t> table, coef;
    frame_rig_layout(B, fmt, hw, h, w, table, coef);
    const int32_t* launch = &table[(size_t)B * H3D_FRAME_RIG_SLOT_WORDS + B];
    memcpy(p->launch, launch, sizeof(p->launch));
    p->host = table;
    p->host.insert(p->host.end(), coef.begin(), coef.end());
    cudaError_t e = cudaSuccess;
    for (int f = 0; f <= H3D_PIXEL_YUYV && e == cudaSuccess; ++f) {   // raise-only, as frame_plan_create does
        if (p->launch[f][H3D_RIG_LAUNCH_SLOTS] == 0) continue;
        cudaFuncAttributes fa;
        const void* kern = rig_kernel_of(f);
        e = cudaFuncGetAttributes(&fa, kern);
        if (e == cudaSuccess && fa.maxDynamicSharedSizeBytes < p->launch[f][H3D_RIG_LAUNCH_SMEM])
            e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, p->launch[f][H3D_RIG_LAUNCH_SMEM]);
    }
    if (e == cudaSuccess) e = cudaMalloc(&p->dev, p->host.size() * 4);
    if (e == cudaSuccess) e = cudaMemcpyAsync(p->dev, p->host.data(), p->host.size() * 4, cudaMemcpyHostToDevice, s);
    if (e != cudaSuccess) {
        cuda_fail(e, "frame_rig_plan_create", __FILE__, __LINE__);
        frame_rig_plan_destroy(p);
        return nullptr;
    }
    p->table = p->dev;
    p->coef = p->dev + table.size();
    return p;
}

void frame_rig_plan_destroy(FrameRigPlan* p) {
    if (!p) return;
    if (p->dev) cudaFree(p->dev);
    delete p;
}

int launch_resize_frames_rig(const FrameRigPlan* p, const uint8_t* const* frames, int normalize, void* out, cudaStream_t s) {
    RigArgs r;
    r.table = p->table; r.coef = p->coef; r.out = out;
    r.B = p->B; r.h = p->h; r.w = p->w; r.normalize = normalize;
    for (int b = 0; b < H3D_FRAME_RIG_MAX_SLOTS; ++b) r.in[b] = b < p->B ? frames[b] : nullptr;
    for (int f = 0; f <= H3D_PIXEL_YUYV; ++f) {
        const int* l = p->launch[f];
        if (l[H3D_RIG_LAUNCH_SLOTS] == 0) continue;
        r.first = l[H3D_RIG_LAUNCH_FIRST]; r.nslots = l[H3D_RIG_LAUNCH_SLOTS];
        const unsigned grid = (unsigned)l[H3D_RIG_LAUNCH_CTAS];
        const int smem = l[H3D_RIG_LAUNCH_SMEM];
        switch (f) {
            case H3D_PIXEL_BGR: resize_frames_rig_kernel<H3D_PIXEL_BGR><<<grid, kFrameThreads, smem, s>>>(r); break;
            case H3D_PIXEL_NV12: resize_frames_rig_kernel<H3D_PIXEL_NV12><<<grid, kFrameThreads, smem, s>>>(r); break;
            case H3D_PIXEL_I420: resize_frames_rig_kernel<H3D_PIXEL_I420><<<grid, kFrameThreads, smem, s>>>(r); break;
            case H3D_PIXEL_YUYV: resize_frames_rig_kernel<H3D_PIXEL_YUYV><<<grid, kFrameThreads, smem, s>>>(r); break;
            default: resize_frames_rig_kernel<H3D_PIXEL_RGB><<<grid, kFrameThreads, smem, s>>>(r); break;
        }
        H3D_CHECK_LAUNCH();
    }
    return H3D_OK;
}

}  // namespace h3d

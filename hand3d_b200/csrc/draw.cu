// Drawing: plot_hand / plot_hand_3d's stick figures (utils/general.py:360-477) as anti-aliased segments rasterised into uint8 RGB
// images in place (h3d_draw_segments; the rule is stated in include/hand3d_b200.h).  This file is compiled with -fmad=false, so that
// every product and sum of the rule is rounded on its own, exactly as a numpy float32 restatement evaluates it.
//
// Work follows the hand, not the frame: the grid is fixed by (B, H, W) (a few CTAs per image), and each CTA strides only over the
// union box of its image's drawable segments.  Each segment's box, expanded by g = h + 1, is part of the rule: a pixel outside it
// gets a = 0.  The extra pixel beyond h makes the box invisible for end points within 2^14 px of the image (d > h outside it after
// rounding too); farther out it keeps a long segment, whose x - c0 and c1 - c0 round alike, from drawing past its end.  Warps walk
// rows, lanes neighbouring pixels; each pixel belongs to one thread, which applies the segments in order, so there are no races.
#include "common.cuh"

namespace h3d {

namespace {

constexpr int kDrawThreads = 256;
constexpr int kDrawWarps = kDrawThreads / 32;
constexpr int kDrawMaxCtas = 64;         // CTAs per image
constexpr int kDrawRowsPerCta = 16;      // an image of H rows gets ceil(H / 16) CTAs, at most kDrawMaxCtas
constexpr int kMaxSeg = H3D_DRAW_MAX_SEGMENTS;

struct DrawArgs {
    uint8_t* images;
    const float* segments;   // [B,S,4]
    const int32_t* valid;    // [B] or nullptr
    int H, W, S, ctas;
    float h;                 // linewidth / 2 + 0.5
    float colors[kMaxSeg * 3];
};

__device__ __forceinline__ float clamp01(float v) { return v > 0.f ? (v < 1.f ? v : 1.f) : 0.f; }   // NaN -> 0

__global__ void __launch_bounds__(kDrawThreads) draw_segments_kernel(const __grid_constant__ DrawArgs a) {
    __shared__ float4 seg[kMaxSeg];      // (r0, c0, r1, c1)
    __shared__ float4 box[kMaxSeg];      // (row lo, row hi, col lo, col hi), expanded by h + 1
    __shared__ float col[kMaxSeg * 3];
    __shared__ int list[kMaxSeg];        // the drawable segments whose box meets the image, in index order
    __shared__ int nlist, y0, y1, x0, x1;
    const int b = blockIdx.x / a.ctas, j = blockIdx.x - b * a.ctas;
    if (a.valid && __ldg(a.valid + b) == 0) return;
    const float g = a.h + 1.f;
    const float Hm = (float)(a.H - 1), Wm = (float)(a.W - 1);
    for (int k = threadIdx.x; k < a.S; k += kDrawThreads) {
        const float* p = a.segments + ((int64_t)b * a.S + k) * 4;
        const float4 s = make_float4(__ldg(p), __ldg(p + 1), __ldg(p + 2), __ldg(p + 3));
        seg[k] = s;
        const bool fin = isfinite(s.x) && isfinite(s.y) && isfinite(s.z) && isfinite(s.w);
        float4 bx = make_float4(fminf(s.x, s.z) - g, fmaxf(s.x, s.z) + g, fminf(s.y, s.w) - g, fmaxf(s.y, s.w) + g);
        if (!fin || bx.y < 0.f || bx.x > Hm || bx.w < 0.f || bx.z > Wm) bx = make_float4(1.f, 0.f, 1.f, 0.f);   // empty
        box[k] = bx;
        col[3 * k] = a.colors[3 * k]; col[3 * k + 1] = a.colors[3 * k + 1]; col[3 * k + 2] = a.colors[3 * k + 2];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int n = 0;
        float ylo = INFINITY, yhi = -INFINITY, xlo = INFINITY, xhi = -INFINITY;
        for (int k = 0; k < a.S; ++k) {
            const float4 bx = box[k];
            if (bx.x > bx.y) continue;
            list[n++] = k;
            ylo = fminf(ylo, bx.x); yhi = fmaxf(yhi, bx.y); xlo = fminf(xlo, bx.z); xhi = fmaxf(xhi, bx.w);
        }
        nlist = n;
        if (n > 0) {   // clipped to the image before the conversion, so that no huge value is converted to int
            y0 = (int)fmaxf(ceilf(ylo), 0.f); y1 = (int)fminf(floorf(yhi), Hm);
            x0 = (int)fmaxf(ceilf(xlo), 0.f); x1 = (int)fminf(floorf(xhi), Wm);
        }
    }
    __syncthreads();
    const int n = nlist;
    if (n == 0) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int rstep = a.ctas * kDrawWarps;
    const int64_t row_bytes = (int64_t)a.W * 3;
    uint8_t* img = a.images + (int64_t)b * a.H * row_bytes;
    for (int y = y0 + j * kDrawWarps + warp; y <= y1; y += rstep) {
        const float fy = (float)y;
        uint8_t* row = img + y * row_bytes;
        for (int x = x0 + lane; x <= x1; x += 32) {
            const float fx = (float)x;
            float v0 = 0.f, v1 = 0.f, v2 = 0.f;
            bool touched = false;
            for (int i = 0; i < n; ++i) {
                const int k = list[i];
                const float4 bx = box[k];
                if (fy < bx.x || fy > bx.y || fx < bx.z || fx > bx.w) continue;
                const float4 s = seg[k];
                const float dy = s.z - s.x, dx = s.w - s.y;
                const float L2 = dy * dy + dx * dx;
                const float ry = fy - s.x, rx = fx - s.y;
                const float t = clamp01(L2 > 0.f ? (ry * dy + rx * dx) / L2 : 0.f);
                const float ey = ry - t * dy, ex = rx - t * dx;
                const float d = sqrtf(ey * ey + ex * ex);
                const float cov = clamp01(a.h - d);
                if (cov > 0.f) {
                    if (!touched) {
                        v0 = (float)row[3 * x]; v1 = (float)row[3 * x + 1]; v2 = (float)row[3 * x + 2];
                        touched = true;
                    }
                    v0 = v0 + cov * (col[3 * k] - v0);
                    v1 = v1 + cov * (col[3 * k + 1] - v1);
                    v2 = v2 + cov * (col[3 * k + 2] - v2);
                }
            }
            if (touched) {
                row[3 * x] = (uint8_t)fminf(fmaxf(rintf(v0), 0.f), 255.f);
                row[3 * x + 1] = (uint8_t)fminf(fmaxf(rintf(v1), 0.f), 255.f);
                row[3 * x + 2] = (uint8_t)fminf(fmaxf(rintf(v2), 0.f), 255.f);
            }
        }
    }
}

}  // namespace

int launch_draw_segments(uint8_t* images, int B, int H, int W, const float* segments, int S, const float* host_colors,
                         const int32_t* valid, float linewidth, cudaStream_t s) {
    DrawArgs a;
    a.images = images; a.segments = segments; a.valid = valid;
    a.H = H; a.W = W; a.S = S;
    a.ctas = std::min(kDrawMaxCtas, ceil_div(H, kDrawRowsPerCta));
    a.h = linewidth / 2.f + 0.5f;
    for (int i = 0; i < kMaxSeg * 3; ++i) a.colors[i] = i < S * 3 ? host_colors[i] : 0.f;
    const int64_t grid = (int64_t)B * a.ctas;
    if (grid >= (1ll << 31)) {
        set_error("h3d_draw_segments: B = %d images of %dx%d is too many for one launch", B, H, W);
        return H3D_EINVAL;
    }
    draw_segments_kernel<<<(unsigned)grid, kDrawThreads, 0, s>>>(a);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

}  // namespace h3d

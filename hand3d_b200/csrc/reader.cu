// Forward generators of the reference's dataset readers, on device (SURVEY.md 8(f) row 4; the training-mode noises of rhd_items and the
// score-map dropout read the per-sample parameters of reader_aug.cu, and are skipped, not applied as identities, when their flag is off):
//   data/BinaryDbReader.py:139-162 palm substitution, :210-250 dominant hand / 21-key-point subsets / root-relative normalisation,
//   :269-346 ground-truth hand crop (centre, size, scale, key-points and intrinsics in crop space), :413-459 score-map targets,
//   data/BinaryDbReaderSTB.py:123-196 (mm -> m, convert_kp, wrist extrapolation), utils/canonical_trafo.py:20-162.
// The image crop itself is crop_image_kernel (h3d_crop_image_from_xy) fed with the centre / scale computed here.
// Arithmetic that feeds comparisons or stored coordinates uses explicit __f*_rn so that nvcc cannot contract to FMA.
#include "common.cuh"

namespace h3d {

// ------------------------------------------------------------------------------------------ RHD items
// One CTA per record.  header [219] = 42x3 xyz | 42x2 uv | 3x3 K; parts [320*320] u8; vis [42] u8.
__global__ void rhd_items_kernel(const float* __restrict__ header, const uint8_t* __restrict__ parts, const uint8_t* __restrict__ vis, int use_wrist,
                                 int hand_crop, int crop_size, float* __restrict__ xyz21, float* __restrict__ uv21, uint8_t* __restrict__ vis21,
                                 float* __restrict__ hand_side, float* __restrict__ kp_scale, float* __restrict__ xyz21_normed,
                                 float* __restrict__ crop_center, float* __restrict__ crop_scale, float* __restrict__ cam_mat,
                                 const float* __restrict__ params, int flags, float* __restrict__ uv42) {
    const int b = blockIdx.x;
    const float* h = header + (int64_t)b * 219;
    __shared__ int s_left, s_right;
    __shared__ float s_xyz[42 * 3], s_uv[42 * 2];
    __shared__ uint8_t s_vis[42];
    if (threadIdx.x == 0) { s_left = 0; s_right = 0; }
    __syncthreads();
    // dominant hand (:212-219): left = part ids 2..17, right = ids > 17
    int nl = 0, nr = 0;
    const uint32_t* p4 = reinterpret_cast<const uint32_t*>(parts + (int64_t)b * 102400);
    for (int i = threadIdx.x; i < 102400 / 4; i += blockDim.x) {
        const uint32_t w = __ldg(p4 + i);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int v = (w >> (8 * j)) & 0xFF;
            nl += (v > 1 && v < 18);
            nr += (v > 17);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { nl += __shfl_xor_sync(0xFFFFFFFFu, nl, o); nr += __shfl_xor_sync(0xFFFFFFFFu, nr, o); }
    if ((threadIdx.x & 31) == 0) { atomicAdd(&s_left, nl); atomicAdd(&s_right, nr); }
    // raw items; uv is cast to int32 and back (:151-154)
    for (int i = threadIdx.x; i < 126; i += blockDim.x) s_xyz[i] = h[i];
    for (int i = threadIdx.x; i < 84; i += blockDim.x) s_uv[i] = (float)(int)h[126 + i];
    for (int i = threadIdx.x; i < 42; i += blockDim.x) s_vis[i] = vis[(int64_t)b * 42 + i] != 0;
    __syncthreads();
    if (threadIdx.x != 0) return;
    if (!use_wrist) {   // palm = mean of key-points 0 and 12 (21 and 33 for the right hand) (:139-162,195-200)
        for (int side = 0; side < 2; ++side) {
            const int a = 21 * side, c = a + 12;
            for (int j = 0; j < 3; ++j) s_xyz[3 * a + j] = __fmul_rn(0.5f, __fadd_rn(s_xyz[3 * a + j], s_xyz[3 * c + j]));
            for (int j = 0; j < 2; ++j) s_uv[2 * a + j] = __fmul_rn(0.5f, __fadd_rn(s_uv[2 * a + j], s_uv[2 * c + j]));
            s_vis[a] = s_vis[a] | s_vis[c];
        }
    }
    const float* prm = params ? params + (int64_t)b * H3D_AUG_PARAMS : nullptr;
    if (flags & H3D_AUG_COORD_UV_NOISE)              // keypoint_uv += truncated_normal([42, 2], 0, 2.5) before the 21-subset (:160-164)
        for (int i = 0; i < 84; ++i) s_uv[i] = __fadd_rn(s_uv[i], prm[H3D_AUG_UV_NOISE + i]);
    if (uv42) for (int i = 0; i < 84; ++i) uv42[(int64_t)b * 84 + i] = s_uv[i];
    const bool left = s_left > s_right;              // 'greater': a tie selects the right hand (:226-231)
    const int o = left ? 0 : 21;
    hand_side[2 * b] = left ? 1.f : 0.f; hand_side[2 * b + 1] = left ? 0.f : 1.f;
    float rel[63];
    for (int k = 0; k < 21; ++k)
        for (int j = 0; j < 3; ++j) {
            const float v = s_xyz[3 * (o + k) + j];
            if (xyz21) xyz21[(int64_t)b * 63 + 3 * k + j] = v;
            rel[3 * k + j] = __fsub_rn(v, s_xyz[3 * o + j]);
        }
    float acc = 0.f;
    for (int j = 0; j < 3; ++j) { const float d = __fsub_rn(rel[36 + j], rel[33 + j]); acc = __fadd_rn(acc, __fmul_rn(d, d)); }
    const float len = sqrtf(acc);                    // index root bone 12 -> 11 (:239-241)
    if (kp_scale) kp_scale[b] = len;
    if (xyz21_normed) for (int i = 0; i < 63; ++i) xyz21_normed[(int64_t)b * 63 + i] = __fdiv_rn(rel[i], len);
    float u[21], v[21];
    for (int k = 0; k < 21; ++k) {
        u[k] = s_uv[2 * (o + k)]; v[k] = s_uv[2 * (o + k) + 1];
        if (vis21) vis21[(int64_t)b * 21 + k] = s_vis[o + k];
    }
    if (hand_crop) {
        float c0 = v[12], c1 = u[12];                // crop centre = key-point 12 as (row, col) (:271)
        if (!(isfinite(c0) && isfinite(c1))) { c0 = 0.f; c1 = 0.f; }
        if (flags & H3D_AUG_CROP_CENTER_NOISE) {     // moves the centre before the crop size is measured (:277-279)
            c0 = __fadd_rn(c0, prm[H3D_AUG_CENTER_NOISE]); c1 = __fadd_rn(c1, prm[H3D_AUG_CENTER_NOISE + 1]);
        }
        const float inf = __int_as_float(0x7f800000);
        float mn0 = inf, mn1 = inf, mx0 = -inf, mx1 = -inf;
        for (int k = 0; k < 21; ++k)
            if (s_vis[o + k]) { mn0 = fminf(mn0, v[k]); mx0 = fmaxf(mx0, v[k]); mn1 = fminf(mn1, u[k]); mx1 = fmaxf(mx1, u[k]); }
        mn0 = fmaxf(mn0, 0.f); mn1 = fmaxf(mn1, 0.f);
        mx0 = fminf(mx0, 320.f); mx1 = fminf(mx1, 320.f);
        float best = fmaxf(__fmul_rn(2.f, fmaxf(__fsub_rn(mx0, c0), __fsub_rn(c0, mn0))), __fmul_rn(2.f, fmaxf(__fsub_rn(mx1, c1), __fsub_rn(c1, mn1))));
        best = fminf(fmaxf(best, 50.f), 500.f);
        if (!isfinite(best)) best = 200.f;
        float sc = __fdiv_rn((float)crop_size, best);
        sc = fminf(fmaxf(sc, 1.f), 10.f);
        if (flags & H3D_AUG_CROP_SCALE_NOISE) sc = __fmul_rn(sc, prm[H3D_AUG_SCALE]);        // scale *= U[1, 1.2) (:307)
        if (flags & H3D_AUG_CROP_OFFSET_NOISE) {     // after the size is fixed: key-points may leave the crop (:310-312)
            c0 = __fadd_rn(c0, prm[H3D_AUG_OFFSET_NOISE]); c1 = __fadd_rn(c1, prm[H3D_AUG_OFFSET_NOISE + 1]);
        }
        if (crop_center) { crop_center[2 * b] = c0; crop_center[2 * b + 1] = c1; }
        if (crop_scale) crop_scale[b] = sc;
        const float half = (float)(crop_size / 2);
        for (int k = 0; k < 21; ++k) {               // key-points in crop space (:325-329)
            u[k] = __fadd_rn(__fmul_rn(__fsub_rn(u[k], c1), sc), half);
            v[k] = __fadd_rn(__fmul_rn(__fsub_rn(v[k], c0), sc), half);
        }
        if (cam_mat) {                               // K' = T S K (:331-358), evaluated as matmul(T, matmul(S, K))
            const float* K = h + 210;
            const float t1 = __fsub_rn(__fmul_rn(c0, sc), half), t2 = __fsub_rn(__fmul_rn(c1, sc), half);
            float SK[9];
            for (int j = 0; j < 3; ++j) { SK[j] = __fmul_rn(sc, K[j]); SK[3 + j] = __fmul_rn(sc, K[3 + j]); SK[6 + j] = K[6 + j]; }
            float* o9 = cam_mat + (int64_t)b * 9;
            for (int j = 0; j < 3; ++j) {
                o9[j] = __fadd_rn(SK[j], __fmul_rn(-t2, SK[6 + j]));
                o9[3 + j] = __fadd_rn(SK[3 + j], __fmul_rn(-t1, SK[6 + j]));
                o9[6 + j] = SK[6 + j];
            }
        }
    } else if (cam_mat) {
        for (int j = 0; j < 9; ++j) cam_mat[(int64_t)b * 9 + j] = h[210 + j];
    }
    if (uv21) for (int k = 0; k < 21; ++k) { uv21[(int64_t)b * 42 + 2 * k] = u[k]; uv21[(int64_t)b * 42 + 2 * k + 1] = v[k]; }
}

int launch_rhd_items(const float* header, const uint8_t* parts, const uint8_t* vis, int B, int use_wrist, int hand_crop, int crop_size,
                     float* xyz21, float* uv21, uint8_t* vis21, float* hand_side, float* kp_scale, float* xyz21_normed, float* crop_center,
                     float* crop_scale, float* cam_mat, cudaStream_t s, const float* params, int flags, float* uv42) {
    H3D_REQUIRE((((uintptr_t)parts) & 3) == 0, "rhd_items: hand_parts must be 4-byte aligned");
    H3D_REQUIRE(params || !(flags & (H3D_AUG_COORD_UV_NOISE | H3D_AUG_CROP_CENTER_NOISE | H3D_AUG_CROP_SCALE_NOISE | H3D_AUG_CROP_OFFSET_NOISE)),
                "rhd_items: noise flags need params");
    rhd_items_kernel<<<B, 256, 0, s>>>(header, parts, vis, use_wrist, hand_crop, crop_size, xyz21, uv21, vis21, hand_side, kp_scale, xyz21_normed,
                                       crop_center, crop_scale, cam_mat, params, flags, uv42);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

// ------------------------------------------------------------------------------------------ STB items
// header [126] = 21x3 xyz (mm) | 21x3 (u, v, valid); convert_kp reorders 0, 20, 19, ..., 1 (data/BinaryDbReaderSTB.py:397-410).
__global__ void stb_items_kernel(const float* __restrict__ header, int B, int use_wrist, float* __restrict__ xyz21, float* __restrict__ uv21,
                                 uint8_t* __restrict__ vis21, float* __restrict__ kp_scale, float* __restrict__ xyz21_normed) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const float* h = header + (int64_t)b * 126;
    float xyz[63], uv[42]; bool vis[21];
    for (int k = 0; k < 21; ++k) {
        const int src = k == 0 ? 0 : 21 - k;
        for (int j = 0; j < 3; ++j) xyz[3 * k + j] = __fdiv_rn(h[3 * src + j], 1000.0f);
        uv[2 * k] = h[63 + 3 * src]; uv[2 * k + 1] = h[63 + 3 * src + 1];
        vis[k] = h[63 + 3 * src + 2] == 1.0f;
    }
    if (use_wrist) {   // wrist = kp16 + 2 (palm - kp16) (:131-134,147-154)
        for (int j = 0; j < 3; ++j) xyz[j] = __fadd_rn(xyz[48 + j], __fmul_rn(2.0f, __fsub_rn(xyz[j], xyz[48 + j])));
        for (int j = 0; j < 2; ++j) uv[j] = __fadd_rn(uv[32 + j], __fmul_rn(2.0f, __fsub_rn(uv[j], uv[32 + j])));
        vis[0] = vis[16] || vis[0];
    }
    float rel[63];
    for (int i = 0; i < 63; ++i) rel[i] = __fsub_rn(xyz[i], xyz[i % 3]);
    float acc = 0.f;
    for (int j = 0; j < 3; ++j) { const float d = __fsub_rn(rel[36 + j], rel[33 + j]); acc = __fadd_rn(acc, __fmul_rn(d, d)); }
    const float len = sqrtf(acc);
    if (kp_scale) kp_scale[b] = len;
    for (int i = 0; i < 63; ++i) {
        if (xyz21) xyz21[(int64_t)b * 63 + i] = xyz[i];
        if (xyz21_normed) xyz21_normed[(int64_t)b * 63 + i] = __fdiv_rn(rel[i], len);
    }
    for (int i = 0; i < 42; ++i) if (uv21) uv21[(int64_t)b * 42 + i] = uv[i];
    for (int k = 0; k < 21; ++k) if (vis21) vis21[(int64_t)b * 21 + k] = vis[k];
}

int launch_stb_items(const float* header, int B, int use_wrist, float* xyz21, float* uv21, uint8_t* vis21, float* kp_scale, float* xyz21_normed,
                     cudaStream_t s) {
    stb_items_kernel<<<ceil_div(B, 64), 64, 0, s>>>(header, B, use_wrist, xyz21, uv21, vis21, kp_scale, xyz21_normed);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

// ------------------------------------------------------------------------------------------ create_multiple_gaussian_map
// out[b, y, x, n] = exp(-((y - r_n)^2 + (x - c_n)^2) / sigma^2) * cond_n with (r_n, c_n) = int32(coords_hw[b, n]) and cond_n = valid_n and
// 0 < r_n < H - 1 and 0 < c_n < W - 1 (data/BinaryDbReader.py:413-459).  HBM-write bound: one thread produces 4 consecutive floats of the
// flattened (x, n) row -> 16-byte stores.
// kDrop: TF 1.3 dropout with one keep bit per (sample, channel) and the reader's rescale, ((g / keep_prob) * bit) * keep_prob, fused
// into the store (data/BinaryDbReader.py:362-365): the per-channel multiply costs no extra traffic.
constexpr int kMaxGaussKp = 64;
template <bool kDrop>
__global__ void gaussian_map_kernel(const float* __restrict__ coords_hw, const uint8_t* __restrict__ valid, int N, int H, int W, float sigma2,
                                    float* __restrict__ out, const float* __restrict__ keep, int keep_stride, float keep_prob) {
    __shared__ float s_r[kMaxGaussKp], s_c[kMaxGaussKp], s_on[kMaxGaussKp], s_keep[kMaxGaussKp];
    const int b = blockIdx.y;
    if (threadIdx.x < N) {
        const int n = threadIdx.x;
        const int r = (int)coords_hw[((int64_t)b * N + n) * 2], c = (int)coords_hw[((int64_t)b * N + n) * 2 + 1];   // tf.cast(float -> int32): truncation
        const bool on = (valid ? valid[(int64_t)b * N + n] != 0 : true) && r < H - 1 && r > 0 && c < W - 1 && c > 0;
        s_r[n] = (float)r; s_c[n] = (float)c; s_on[n] = on ? 1.f : 0.f;
        if (kDrop) s_keep[n] = keep[(int64_t)b * keep_stride + n];
    }
    __syncthreads();
    const int row_elems = W * N;                     // multiple of 4 is required by the launcher
    const int vec_per_row = row_elems >> 2;
    const int64_t total = (int64_t)H * vec_per_row;
    float* ob = out + (int64_t)b * H * row_elems;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int y = (int)(i / vec_per_row), v = (int)(i - (int64_t)y * vec_per_row);
        float o4[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int e = 4 * v + j;
            const int x = e / N, n = e - x * N;
            const float dy = __fsub_rn((float)y, s_r[n]), dx = __fsub_rn((float)x, s_c[n]);
            const float dist = __fadd_rn(__fmul_rn(dy, dy), __fmul_rn(dx, dx));
            o4[j] = __fmul_rn(expf(__fdiv_rn(-dist, sigma2)), s_on[n]);
            if (kDrop) o4[j] = __fmul_rn(__fmul_rn(__fdiv_rn(o4[j], keep_prob), s_keep[n]), keep_prob);
        }
        reinterpret_cast<float4*>(ob)[i] = make_float4(o4[0], o4[1], o4[2], o4[3]);
    }
}

int launch_gaussian_map(const float* coords_hw, const uint8_t* valid, int B, int N, int H, int W, float sigma, float* out, cudaStream_t s,
                        const float* keep, int keep_stride, float keep_prob) {
    H3D_REQUIRE(N >= 1 && N <= kMaxGaussKp && ((W * N) & 3) == 0, "gaussian_scoremap: N must be in [1,64] and W * N a multiple of 4");
    H3D_REQUIRE(!keep || (keep_stride >= N && keep_prob > 0.f && keep_prob <= 1.f), "gaussian_scoremap: keep_stride < N or keep_prob outside (0, 1]");
    const int64_t total = (int64_t)H * (W * N / 4);
    dim3 grid((unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div64(total, 256), 132 * 8 / std::max(1, std::min(B, 8)))), B);
    if (keep) gaussian_map_kernel<true><<<grid, 256, 0, s>>>(coords_hw, valid, N, H, W, sigma * sigma, out, keep, keep_stride, keep_prob);
    else gaussian_map_kernel<false><<<grid, 256, 0, s>>>(coords_hw, valid, N, H, W, sigma * sigma, out, nullptr, 0, 1.f);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

// ------------------------------------------------------------------------------------------ canonical_trafo
// utils/canonical_trafo.py:20-136 (+ flip_right_hand :139-162, + tf.matrix_inverse of the total rotation as the readers store it).
__device__ __forceinline__ float atan2_ref(float y, float x) {
    const float pi = 3.141592653589793f;
    const float xe = __fadd_rn(x, 1e-8f);
    float t = atanf(__fdiv_rn(y, xe));
    if (xe < 0.f) t = __fadd_rn(t, pi);
    if (t < 0.f) t = __fadd_rn(t, __fmul_rn(2.f, pi));
    if (t > pi) t = __fadd_rn(t, __fmul_rn(-2.f, pi));
    return t;
}
__device__ __forceinline__ void mat3_mul(const float* a, const float* b, float* c) {     // c = a b, separate multiply / add
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            c[3 * i + j] = __fadd_rn(__fadd_rn(__fmul_rn(a[3 * i], b[j]), __fmul_rn(a[3 * i + 1], b[3 + j])), __fmul_rn(a[3 * i + 2], b[6 + j]));
}
__device__ __forceinline__ void pts_mul(float* p, const float* m) {                      // p[21,3] <- p m
    for (int k = 0; k < 21; ++k) {
        const float x = p[3 * k], y = p[3 * k + 1], z = p[3 * k + 2];
        for (int j = 0; j < 3; ++j) p[3 * k + j] = __fadd_rn(__fadd_rn(__fmul_rn(x, m[j]), __fmul_rn(y, m[3 + j])), __fmul_rn(z, m[6 + j]));
    }
}
__global__ void canonical_trafo_kernel(const float* __restrict__ xyz, const uint8_t* __restrict__ cond_right, int B, float* __restrict__ can,
                                       float* __restrict__ rot, float* __restrict__ rot_inv) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    float p[63];
    for (int i = 0; i < 63; ++i) p[i] = __fsub_rn(xyz[(int64_t)b * 63 + i], xyz[(int64_t)b * 63 + i % 3]);
    float total[9], r[9], tmp[9];
    {   // rotate the middle-finger root into the yz plane
        const float a = atan2_ref(p[36], p[37]);
        const float c = cosf(a), s = sinf(a);
        const float m[9] = {c, s, 0.f, -s, c, 0.f, 0.f, 0.f, 1.f};
        for (int i = 0; i < 9; ++i) total[i] = m[i];
        pts_mul(p, m);
    }
    {   // ... and onto the y axis
        const float beta = -atan2_ref(p[38], p[37]);
        const float a = __fadd_rn(beta, 3.141592653589793f);
        const float c = cosf(a), s = sinf(a);
        const float m[9] = {1.f, 0.f, 0.f, 0.f, c, s, 0.f, -s, c};
        for (int i = 0; i < 9; ++i) r[i] = m[i];
        pts_mul(p, r);
        mat3_mul(total, r, tmp);
        for (int i = 0; i < 9; ++i) total[i] = tmp[i];
    }
    {   // fix the rotation about y with the pinky root
        const float a = atan2_ref(p[62], p[60]);
        const float c = cosf(a), s = sinf(a);
        const float m[9] = {c, 0.f, -s, 0.f, 1.f, 0.f, s, 0.f, c};
        for (int i = 0; i < 9; ++i) r[i] = m[i];
        pts_mul(p, r);
        mat3_mul(total, r, tmp);
        for (int i = 0; i < 9; ++i) total[i] = tmp[i];
    }
    const bool flip = cond_right && cond_right[b];
    if (can) for (int i = 0; i < 63; ++i) can[(int64_t)b * 63 + i] = (flip && (i % 3) == 2) ? -p[i] : p[i];
    if (rot) for (int i = 0; i < 9; ++i) rot[(int64_t)b * 9 + i] = total[i];
    if (rot_inv) {   // general 3x3 inverse (adjugate / determinant), as tf.matrix_inverse is applied to the product
        const float* m = total;
        const float c00 = m[4] * m[8] - m[5] * m[7], c01 = m[5] * m[6] - m[3] * m[8], c02 = m[3] * m[7] - m[4] * m[6];
        const float det = m[0] * c00 + m[1] * c01 + m[2] * c02;
        const float id = 1.0f / det;
        float* o = rot_inv + (int64_t)b * 9;
        o[0] = c00 * id; o[1] = (m[2] * m[7] - m[1] * m[8]) * id; o[2] = (m[1] * m[5] - m[2] * m[4]) * id;
        o[3] = c01 * id; o[4] = (m[0] * m[8] - m[2] * m[6]) * id; o[5] = (m[2] * m[3] - m[0] * m[5]) * id;
        o[6] = c02 * id; o[7] = (m[1] * m[6] - m[0] * m[7]) * id; o[8] = (m[0] * m[4] - m[1] * m[3]) * id;
    }
}

int launch_canonical_trafo(const float* xyz, const uint8_t* cond_right, int B, float* can, float* rot, float* rot_inv, cudaStream_t s) {
    canonical_trafo_kernel<<<ceil_div(B, 64), 64, 0, s>>>(xyz, cond_right, B, can, rot, rot_inv);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

}  // namespace h3d

// Training kernels of the lifting stage (training_lifting.py): the adjoints of the Rodrigues rotation + right-hand flip + rotate that
// ends the 'proposed' variant and of the forward kinematics of the 'local*' variants, the forward analysis bone_rel_trafo that builds
// the 'local' target, and the mean squared error every variant's loss is made of.
//
// Conventions (as train.cu): every launcher only enqueues (scratch is the caller's), nothing synchronises, no float atomics, and
// every sum runs in an order fixed by the shapes alone, so results are bit-reproducible and a training step can be captured into a
// CUDA graph.
#include "common.cuh"

namespace h3d {

namespace {

constexpr int kMseThreads = 256;
constexpr float kPi = 3.141592653589793f;

// =============================================================================================
// Adjoint of rotate_canonical_kernel (elementwise.cu): R = rodrigues(u), c' = flip_z(can) where argmax(hand_side) == 1,
// out = c' R.  One block of 64 threads per sample:
//   d_can[k, i] = s_i sum_j d_out[k, j] R[i, j]                (s_2 = -1 for a right hand)
//   G[i, j]     = d_R[i, j] + sum_k c'[k, i] d_out[k, j]       (k ascending)
// and thread 0 takes G back through R = ct I + (1 - ct) n n^T + st [n]_x, n = u / theta, theta = sqrt(|u|^2 + 1e-8) (DESIGN 4.9).
// =============================================================================================
__global__ void __launch_bounds__(64) rotate_canonical_backward_kernel(const float* __restrict__ can, const float* __restrict__ uxyz,
                                                                       const float* __restrict__ hand_side, const float* __restrict__ d_out,
                                                                       const float* __restrict__ d_R, float* __restrict__ d_can,
                                                                       float* __restrict__ d_uxyz) {
    const int b = blockIdx.x, t = threadIdx.x;
    __shared__ float R[9], G[9];
    const float ub[3] = {__ldg(uxyz + 3 * b), __ldg(uxyz + 3 * b + 1), __ldg(uxyz + 3 * b + 2)};
    if (t == 0) rodrigues_rot_mat(ub[0], ub[1], ub[2], R);
    __syncthreads();
    const bool right = hand_side[2 * b + 1] > hand_side[2 * b];   // as the forward: argmax(hand_side, 1) == 1, ties -> index 0
    const float* cb = can + 63 * b;
    const float* ob = d_out ? d_out + 63 * b : nullptr;
    if (t < 63) {
        const int k = t / 3, i = t - 3 * (t / 3);
        float acc = 0.f;
        if (ob) {
            for (int j = 0; j < 3; ++j) acc = __fadd_rn(acc, __fmul_rn(__ldg(ob + 3 * k + j), R[3 * i + j]));
            if (right && i == 2) acc = -acc;
        }
        d_can[63 * b + t] = acc;
    }
    if (t < 9) {
        const int i = t / 3, j = t - 3 * (t / 3);
        float g = d_R ? __ldg(d_R + 9 * b + t) : 0.f;
        if (ob) {
            float acc = 0.f;
            for (int k = 0; k < 21; ++k) {
                float c = __ldg(cb + 3 * k + i);
                if (right && i == 2) c = -c;
                acc = __fadd_rn(acc, __fmul_rn(c, __ldg(ob + 3 * k + j)));
            }
            g = __fadd_rn(g, acc);
        }
        G[t] = g;
    }
    __syncthreads();
    if (t != 0) return;
    // the forward's scalars, from its own fp32 operations (rodrigues_rot_mat)
    const float n2 = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(ub[0], ub[0]), __fmul_rn(ub[1], ub[1])), __fmul_rn(ub[2], ub[2])), 1e-8f);
    const float theta = sqrtf(n2);
    const float st = sinf(theta), ct = cosf(theta);
    const float one_ct = __fsub_rn(1.0f, ct);
    const float nf = __fdiv_rn(1.0f, theta);
    const float n[3] = {__fmul_rn(ub[0], nf), __fmul_rn(ub[1], nf), __fmul_rn(ub[2], nf)};
    // R[i][j] = ct delta_ij + one_ct n_i n_j + st E_ij, E = [n]_x = [[0,-nz,ny],[nz,0,-nx],[-ny,nx,0]]
    const float d_ct = G[0] + G[4] + G[8];
    float d_one_ct = 0.f;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) d_one_ct += G[3 * i + j] * n[i] * n[j];
    const float e[3] = {G[7] - G[5], G[2] - G[6], G[3] - G[1]};   // d R / d(st n_i) contracted with G
    const float d_st = e[0] * n[0] + e[1] * n[1] + e[2] * n[2];
    float d_n[3];
    for (int i = 0; i < 3; ++i) {
        float s = 0.f;
        for (int j = 0; j < 3; ++j) s += (G[3 * i + j] + G[3 * j + i]) * n[j];
        d_n[i] = one_ct * s + st * e[i];
    }
    // theta enters through sin, cos and nf = 1 / theta;  theta = sqrt(n2), d n2 / d u_i = 2 u_i
    const float d_nf = d_n[0] * ub[0] + d_n[1] * ub[1] + d_n[2] * ub[2];
    const float d_theta = (d_one_ct - d_ct) * st + d_st * ct - d_nf * nf * nf;
    const float k = d_theta * nf;                                   // d_theta / (2 theta) * 2
    for (int i = 0; i < 3; ++i) d_uxyz[3 * b + i] = d_n[i] * nf + k * ub[i];
}

// =============================================================================================
// Forward kinematics (bone_rel_trafo_inv_kernel, elementwise.cu) and its adjoint.  Per chain step, with the reference's
// T <- Trans_z(-len) RotX(-ax) RotY(-ay) T written as R <- M R, t <- M t - len e_z (M = RotX(a) RotY(b), a = -angle_x, b = -angle_y),
// and the key-point x = -R^T t.  One thread per (sample, chain): the root and the five fingers are independent chains of 1 and 4 bones.
// =============================================================================================
struct Rig { float R[9], t[3]; };

__device__ __forceinline__ void rot_xy(float a, float bb, float* M) {   // M = RotX(a) RotY(bb)
    const float cx = cosf(a), sx = sinf(a), cy = cosf(bb), sy = sinf(bb);
    M[0] = cy; M[1] = 0.f; M[2] = sy;
    M[3] = sx * sy; M[4] = cx; M[5] = -sx * cy;
    M[6] = -cx * sy; M[7] = sx; M[8] = cx * cy;
}

__device__ __forceinline__ void rig_step(Rig& g, const float* M, float len) {
    Rig o;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int j = 0; j < 3; ++j) o.R[3 * i + j] = M[3 * i] * g.R[j] + M[3 * i + 1] * g.R[3 + j] + M[3 * i + 2] * g.R[6 + j];
        o.t[i] = M[3 * i] * g.t[0] + M[3 * i + 1] * g.t[1] + M[3 * i + 2] * g.t[2];
    }
    o.t[2] -= len;
    g = o;
}

__device__ __forceinline__ int chain_bone(int c, int i) { return c == 0 ? 0 : 4 * c - i; }   // kinematic_chain_list order

__global__ void bone_rel_trafo_inv_backward_kernel(const float* __restrict__ rel, const float* __restrict__ d_xyz,
                                                   float* __restrict__ d_rel, int B) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= B * 6) return;
    const int b = idx / 6, c = idx - b * 6;
    const int n = c == 0 ? 1 : 4;
    // forward, keeping the rig before each step (at most four steps, all indices compile-time after unrolling)
    Rig st[4];
    Rig g;
#pragma unroll
    for (int j = 0; j < 9; ++j) g.R[j] = (j % 4 == 0) ? 1.f : 0.f;
    g.t[0] = g.t[1] = g.t[2] = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        if (i < n) {
            st[i] = g;
            const float* r = rel + ((int64_t)b * 21 + chain_bone(c, i)) * 3;
            float M[9];
            rot_xy(-r[1], -r[2], M);
            rig_step(g, M, r[0]);
        }
    }
    // reverse: dR, dt are the adjoints of the rig after step i
    float dR[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, dt[3] = {0, 0, 0};
#pragma unroll
    for (int i = 3; i >= 0; --i) {
        if (i >= n) continue;
        const int bone = chain_bone(c, i);
        const float* r = rel + ((int64_t)b * 21 + bone) * 3;
        const float* gx = d_xyz + ((int64_t)b * 21 + bone) * 3;
        const float g0 = gx[0], g1 = gx[1], g2 = gx[2];
        // x_j = -sum_m R[m][j] t[m] of the rig after step i (= g)
#pragma unroll
        for (int m = 0; m < 3; ++m) {
            dR[3 * m + 0] -= g0 * g.t[m];
            dR[3 * m + 1] -= g1 * g.t[m];
            dR[3 * m + 2] -= g2 * g.t[m];
            dt[m] -= g.R[3 * m] * g0 + g.R[3 * m + 1] * g1 + g.R[3 * m + 2] * g2;
        }
        const Rig& p = st[i];
        const float a = -r[1], bb = -r[2];
        const float cx = cosf(a), sx = sinf(a), cy = cosf(bb), sy = sinf(bb);
        float M[9];
        rot_xy(a, bb, M);
        // dM[a][c] = sum_j dR[a][j] p.R[c][j] + dt[a] p.t[c]
        float dM[9];
#pragma unroll
        for (int u = 0; u < 3; ++u)
#pragma unroll
            for (int v = 0; v < 3; ++v)
                dM[3 * u + v] = dR[3 * u] * p.R[3 * v] + dR[3 * u + 1] * p.R[3 * v + 1] + dR[3 * u + 2] * p.R[3 * v + 2] + dt[u] * p.t[v];
        const float d_len = -dt[2];
        const float d_a = dM[3] * (cx * sy) - dM[4] * sx - dM[5] * (cx * cy) + dM[6] * (sx * sy) + dM[7] * cx - dM[8] * (sx * cy);
        const float d_b = -dM[0] * sy + dM[2] * cy + dM[3] * (sx * cy) + dM[5] * (sx * sy) - dM[6] * (cx * cy) - dM[8] * (cx * sy);
        float* o = d_rel + ((int64_t)b * 21 + bone) * 3;
        o[0] = d_len; o[1] = -d_a; o[2] = -d_b;
        // to the rig before step i: R = M R_p, t = M t_p - len e_z
        float nR[9], nt[3];
#pragma unroll
        for (int u = 0; u < 3; ++u) {
#pragma unroll
            for (int v = 0; v < 3; ++v) nR[3 * u + v] = M[u] * dR[v] + M[3 + u] * dR[3 + v] + M[6 + u] * dR[6 + v];
            nt[u] = M[u] * dt[0] + M[3 + u] * dt[1] + M[6 + u] * dt[2];
        }
#pragma unroll
        for (int j = 0; j < 9; ++j) dR[j] = nR[j];
#pragma unroll
        for (int j = 0; j < 3; ++j) dt[j] = nt[j];
        g = p;
    }
}

// =============================================================================================
// bone_rel_trafo (utils/relative_trafo.py:184-240): xyz -> (length, angle_x, angle_y) per bone, with the reference's own atan2
// (:27-46: atan(y / (x + 1e-8)) and its quadrant corrections, in fp32 as TF evaluates them).
// =============================================================================================
__device__ __forceinline__ float atan2_ref(float y, float x) {
    const float xe = __fadd_rn(x, 1e-8f);
    float a = atanf(__fdiv_rn(y, xe));
    a = __fadd_rn(a, xe < 0.f ? kPi : 0.f);
    a = __fadd_rn(a, a < 0.f ? 2.f * kPi : 0.f);
    return __fadd_rn(a, a > kPi ? -2.f * kPi : 0.f);
}

__global__ void bone_rel_trafo_kernel(const float* __restrict__ xyz, float* __restrict__ rel, int B) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= B * 6) return;
    const int b = idx / 6, c = idx - b * 6;
    const int n = c == 0 ? 1 : 4;
    const float* xb = xyz + (int64_t)b * 63;
    Rig g;
    for (int j = 0; j < 9; ++j) g.R[j] = (j % 4 == 0) ? 1.f : 0.f;
    g.t[0] = g.t[1] = g.t[2] = 0.f;
    int parent = -1;
    for (int i = 0; i < n; ++i) {
        const int bone = chain_bone(c, i);
        float d[3];
        if (parent < 0) {
            d[0] = xb[3 * bone]; d[1] = xb[3 * bone + 1]; d[2] = xb[3 * bone + 2];
        } else {   // T x_child - T x_parent, both in the parent's frame
            for (int m = 0; m < 3; ++m) {
                const float xc = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(g.R[3 * m], xb[3 * bone]), __fmul_rn(g.R[3 * m + 1], xb[3 * bone + 1])),
                                                     __fmul_rn(g.R[3 * m + 2], xb[3 * bone + 2])), g.t[m]);
                const float xp = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(g.R[3 * m], xb[3 * parent]), __fmul_rn(g.R[3 * m + 1], xb[3 * parent + 1])),
                                                     __fmul_rn(g.R[3 * m + 2], xb[3 * parent + 2])), g.t[m]);
                d[m] = __fsub_rn(xc, xp);
            }
        }
        const float len = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2])));
        const float ay = atan2_ref(d[0], d[2]);
        // RotY(-ay) d: its y row keeps d[1], its z row is sin(ay) d[0] + cos(ay) d[2]
        const float tz = __fadd_rn(__fmul_rn(sinf(ay), d[0]), __fmul_rn(cosf(ay), d[2]));
        const float ax = atan2_ref(-d[1], tz);
        float* o = rel + ((int64_t)b * 21 + bone) * 3;
        o[0] = len; o[1] = ax; o[2] = ay;
        float M[9];
        rot_xy(-ax, -ay, M);
        rig_step(g, M, len);
        parent = bone;
    }
}

// =============================================================================================
// Mean squared error reduce_mean(square(p - t)) over n elements: per-block partial sums (thread-strided, then a fixed tree), one
// finalising block; the gradient is (g / n) (2 (p - t)), as TF's MeanGrad and SquareGrad evaluate it.
// =============================================================================================
__device__ float tree_sum(float* red, float v) {
    const int t = threadIdx.x;
    red[t] = v;
    __syncthreads();
    for (int h = kMseThreads / 2; h > 0; h >>= 1) {
        if (t < h) red[t] = __fadd_rn(red[t], red[t + h]);
        __syncthreads();
    }
    return red[0];
}

__global__ void __launch_bounds__(kMseThreads) mse_partial_kernel(const float* __restrict__ p, const float* __restrict__ q,
                                                                  float* __restrict__ partial, int64_t n, int64_t per_block) {
    __shared__ float red[kMseThreads];
    const int64_t i0 = (int64_t)blockIdx.x * per_block, i1 = min(n, i0 + per_block);
    float s = 0.f;
    for (int64_t i = i0 + threadIdx.x; i < i1; i += kMseThreads) {
        const float d = __fsub_rn(__ldg(p + i), __ldg(q + i));
        s = __fadd_rn(s, __fmul_rn(d, d));
    }
    const float tot = tree_sum(red, s);
    if (threadIdx.x == 0) partial[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(kMseThreads) mse_finalize_kernel(const float* __restrict__ partial, int nblk, float* __restrict__ loss,
                                                                   int64_t n) {
    __shared__ float red[kMseThreads];
    float s = 0.f;
    for (int i = threadIdx.x; i < nblk; i += kMseThreads) s = __fadd_rn(s, partial[i]);
    const float tot = tree_sum(red, s);
    if (threadIdx.x == 0) *loss = __fdiv_rn(tot, (float)n);
}

__global__ void mse_grad_kernel(const float* __restrict__ p, const float* __restrict__ q, const float* __restrict__ grad,
                                float* __restrict__ dp, int64_t n) {
    const float gn = __fdiv_rn(grad ? __ldg(grad) : 1.f, (float)n);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        dp[i] = __fmul_rn(gn, __fmul_rn(2.f, __fsub_rn(__ldg(p + i), __ldg(q + i))));
}

// Blocks of the MSE reduction: at most 1024, at least 2048 elements each (shape-only policy, as the cross-entropy's)
int mse_blocks(int64_t n, int64_t* per_block) {
    const int64_t nblk = std::max<int64_t>(1, std::min<int64_t>(ceil_div64(n, 2048), 1024));
    *per_block = ceil_div64(n, nblk);
    return (int)ceil_div64(n, *per_block);
}

}  // namespace

int launch_rotate_canonical_backward(const float* can, const float* uxyz, const float* hand_side, const float* d_out, const float* d_R,
                                     int B, float* d_can, float* d_uxyz, cudaStream_t s) {
    rotate_canonical_backward_kernel<<<B, 64, 0, s>>>(can, uxyz, hand_side, d_out, d_R, d_can, d_uxyz);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

int launch_bone_rel_trafo_inv_backward(const float* rel, const float* d_xyz, float* d_rel, int B, cudaStream_t s) {
    bone_rel_trafo_inv_backward_kernel<<<ceil_div(B * 6, 128), 128, 0, s>>>(rel, d_xyz, d_rel, B);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

int launch_bone_rel_trafo(const float* xyz, float* rel, int B, cudaStream_t s) {
    bone_rel_trafo_kernel<<<ceil_div(B * 6, 128), 128, 0, s>>>(xyz, rel, B);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

int64_t mse_scratch_floats(int64_t n) { int64_t pb; return mse_blocks(n, &pb); }

int launch_mse(const float* p, const float* q, float* scratch, int64_t n, float* loss, cudaStream_t s) {
    int64_t pb = 0;
    const int nblk = mse_blocks(n, &pb);
    mse_partial_kernel<<<nblk, kMseThreads, 0, s>>>(p, q, scratch, n, pb);
    H3D_CHECK_LAUNCH();
    mse_finalize_kernel<<<1, kMseThreads, 0, s>>>(scratch, nblk, loss, n);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

int launch_mse_grad(const float* p, const float* q, const float* grad, float* dp, int64_t n, cudaStream_t s) {
    const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div64(n, 256 * 4), 132 * 32));
    mse_grad_kernel<<<blocks, 256, 0, s>>>(p, q, grad, dp, n);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

}  // namespace h3d

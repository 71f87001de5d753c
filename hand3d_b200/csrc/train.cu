// Training kernels of HandSegNet and PoseNet2D (training_posenet.py, training_handsegnet.py): the gradient of the TF1-legacy bilinear
// resize that sits between each network and its loss, the two training losses with their gradients, and TF 1.3's Adam step.
//
// Conventions (as conv_wgrad.cu): every launcher only enqueues (scratch is the caller's), nothing synchronises, so a whole training
// step can be captured into a CUDA graph; no float atomics, and every sum runs in an order fixed by the shapes alone, so results are
// bit-reproducible run to run.  Arithmetic that TF evaluates as separate operations uses explicit __f*_rn so that nvcc cannot
// contract it into FMAs.
#include "common.cuh"

namespace h3d {

namespace {

constexpr int kRedThreads = 256;   // block size of every fixed-order reduction below

// Sum of a[0..n) by one block of kRedThreads threads: strided partial sums in index order, then a fixed tree in shared memory.
// Every thread returns the total.  The order depends on n only, so two kernels calling it on the same data agree bit for bit.
__device__ float block_sum_fixed(const float* __restrict__ a, int n, float* red) {
    const int t = threadIdx.x;
    float s = 0.f;
    for (int i = t; i < n; i += kRedThreads) s = __fadd_rn(s, __ldg(a + i));
    red[t] = s;
    __syncthreads();
    for (int h = kRedThreads / 2; h > 0; h >>= 1) {
        if (t < h) red[t] = __fadd_rn(red[t], red[t + h]);
        __syncthreads();
    }
    const float r = red[0];
    __syncthreads();
    return r;
}

// Fixed tree over red[0..kRedThreads) written by the caller; returns the total in every thread.
__device__ float block_tree(float* red) {
    const int t = threadIdx.x;
    __syncthreads();
    for (int h = kRedThreads / 2; h > 0; h >>= 1) {
        if (t < h) red[t] = __fadd_rn(red[t], red[t + h]);
        __syncthreads();
    }
    const float r = red[0];
    __syncthreads();
    return r;
}

// =============================================================================================
// Gradient of tf.image.resize_images (bilinear, align_corners=False, TF1 legacy): the adjoint of resize_bilinear_tf1_kernel
// (elementwise.cu).  Separable, so it runs as two 1-D transposed passes, each a GATHER: input index i of the pass sums, over the
// candidate output indices o in ascending order, g[o] (1 - l(o)) where i0(o) == i and g[o] l(o) where i1(o) == i.  i0, i1 and l are
// recomputed with the forward's own fp32 operations (in = o * scale, floorf, min(i0 + 1, n - 1), in - i0), so a clamped edge
// receives both weights exactly as the forward reads it.  The candidate range only has to contain every contributing o; it is
// widened by two on each side and every candidate is checked, so float rounding of the ratio cannot drop a term.
// =============================================================================================
struct Src1d { int i0, i1; float l; };
__device__ __forceinline__ Src1d src_1d(int o, float scale, int n) {
    const float in = __fmul_rn((float)o, scale);
    Src1d s;
    s.i0 = (int)floorf(in);
    s.i1 = min(s.i0 + 1, n - 1);
    s.l = __fsub_rn(in, (float)s.i0);
    return s;
}

// Range of output indices o (of `out`) that may read input index i (of `in`): in(o) in [i - 1, i + 1), with two indices of margin.
__device__ __forceinline__ void cand_range(int i, int in, int out, int* lo, int* hi) {
    const int64_t a = (int64_t)(i - 1) * out, b = (int64_t)(i + 1) * out;
    *lo = max(0, (int)(a >= 0 ? a / in : -((-a + in - 1) / in)) - 2);
    *hi = min(out - 1, (int)((b + in - 1) / in) + 2);
}

// Columns: t[b, oy, xi, c] = sum_ox dy[b, oy, ox, c] w_x(ox -> xi);  dy [B, rows, ow, C] -> t [B, rows, W, C]
template <int CT>
__global__ void resize_grad_cols_kernel(const float* __restrict__ dy, float* __restrict__ t, int64_t BR, int W, int ow, int C_rt,
                                        float wscale) {
    const int C = CT > 0 ? CT : C_rt;
    const int64_t total = BR * W * C;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const int xi = (int)((i / C) % W);
        const int64_t r = i / ((int64_t)C * W);
        const float* src = dy + r * ow * C + c;
        int lo, hi;
        cand_range(xi, W, ow, &lo, &hi);
        float acc = 0.f;
        for (int ox = lo; ox <= hi; ++ox) {
            const Src1d s = src_1d(ox, wscale, W);
            if (s.i0 == xi || s.i1 == xi) {
                const float g = __ldg(src + (int64_t)ox * C);
                if (s.i0 == xi) acc = __fadd_rn(acc, __fmul_rn(g, __fsub_rn(1.f, s.l)));
                if (s.i1 == xi) acc = __fadd_rn(acc, __fmul_rn(g, s.l));
            }
        }
        t[i] = acc;
    }
}

// Rows: dx[b, yi, x, c] = sum_oy t[b, oy, x, c] w_y(oy -> yi);  t [B, oh, RW] -> dx [B, H, RW] (RW = W * C floats per row)
__global__ void resize_grad_rows_kernel(const float* __restrict__ t, float* __restrict__ dx, int B, int H, int oh, int64_t RW, float hscale) {
    const int64_t total = (int64_t)B * H * RW;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t e = i % RW;
        const int yi = (int)((i / RW) % H);
        const int b = (int)(i / (RW * H));
        const float* src = t + (int64_t)b * oh * RW + e;
        int lo, hi;
        cand_range(yi, H, oh, &lo, &hi);
        float acc = 0.f;
        for (int oy = lo; oy <= hi; ++oy) {
            const Src1d s = src_1d(oy, hscale, H);
            if (s.i0 == yi || s.i1 == yi) {
                const float g = __ldg(src + (int64_t)oy * RW);
                if (s.i0 == yi) acc = __fadd_rn(acc, __fmul_rn(g, __fsub_rn(1.f, s.l)));
                if (s.i1 == yi) acc = __fadd_rn(acc, __fmul_rn(g, s.l));
            }
        }
        dx[i] = acc;
    }
}

// =============================================================================================
// PoseNet score-map loss (training_posenet.py:58-61) for one predicted map:
//   L = sum_{b,k} vis[b,k] sqrt(mean_{h,w} (P - T)^2) / (sum_{b,k} vis + 0.001)
// =============================================================================================
constexpr int kSmK = 21, kSmGroups = 12, kSmThreads = kSmK * kSmGroups;   // 252 threads: thread t = (pixel group t / 21, channel t % 21)

// partial[b][chunk][k] = sum over the chunk's pixels (group-strided, then the 12 groups in order) of (P - T)^2
__global__ void __launch_bounds__(kSmThreads) scoremap_sq_partial_kernel(const float* __restrict__ P, const float* __restrict__ T,
                                                                          float* __restrict__ partial, int HW, int ppc, int nchunk) {
    __shared__ float red[kSmGroups][kSmK];
    const int b = blockIdx.y, chunk = blockIdx.x, t = threadIdx.x, k = t % kSmK, j = t / kSmK;
    const int p0 = chunk * ppc, p1 = min(HW, p0 + ppc);
    const int64_t base = (int64_t)b * HW * kSmK;
    float s = 0.f;
    for (int p = p0 + j; p < p1; p += kSmGroups) {
        const int64_t o = base + (int64_t)p * kSmK + k;
        const float d = __fsub_rn(__ldg(P + o), __ldg(T + o));
        s = __fadd_rn(s, __fmul_rn(d, d));
    }
    red[j][k] = s;
    __syncthreads();
    if (j == 0) {
        float r = red[0][k];
        for (int g = 1; g < kSmGroups; ++g) r = __fadd_rn(r, red[g][k]);
        partial[((int64_t)b * nchunk + chunk) * kSmK + k] = r;
    }
}

// rms[b,k] = sqrt(sum_chunks partial / HW) in chunk order; loss = sum vis rms / (sum vis + 0.001); one block of kRedThreads
__global__ void __launch_bounds__(kRedThreads) scoremap_loss_finalize_kernel(const float* __restrict__ partial, const float* __restrict__ vis,
                                                                             float* __restrict__ rms, float* __restrict__ loss, int n, int HW,
                                                                             int nchunk) {
    __shared__ float red[kRedThreads];
    const int t = threadIdx.x;
    float wsum = 0.f;
    for (int i = t; i < n; i += kRedThreads) {
        const int b = i / kSmK, k = i % kSmK;
        const float* src = partial + (int64_t)b * nchunk * kSmK + k;
        float ss = 0.f;
        for (int c = 0; c < nchunk; ++c) ss = __fadd_rn(ss, src[(int64_t)c * kSmK]);
        const float r = __fsqrt_rn(__fdiv_rn(ss, (float)HW));
        rms[i] = r;
        wsum = __fadd_rn(wsum, __fmul_rn(__ldg(vis + i), r));
    }
    red[t] = wsum;
    const float num = block_tree(red);
    const float S = __fadd_rn(block_sum_fixed(vis, n, red), 0.001f);
    if (t == 0) *loss = __fdiv_rn(num, S);
}

// dP = g vis[b,k] / S (P - T) / (HW rms[b,k]); 0 where rms == 0 (TF: SqrtGrad's inf times 0 gives NaN there)
__global__ void __launch_bounds__(kRedThreads) scoremap_loss_grad_kernel(const float* __restrict__ P, const float* __restrict__ T,
                                                                         const float* __restrict__ vis, const float* __restrict__ rms,
                                                                         const float* __restrict__ grad, float* __restrict__ dP, int n,
                                                                         int HW) {
    __shared__ float red[kRedThreads];
    const float S = __fadd_rn(block_sum_fixed(vis, n, red), 0.001f);
    const float g = grad ? __ldg(grad) : 1.f;
    const int64_t total = (int64_t)n * HW;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int k = (int)(i % kSmK);
        const int b = (int)(i / ((int64_t)HW * kSmK));
        const int bk = b * kSmK + k;
        const float r = __ldg(rms + bk);
        float coef = 0.f;
        if (r != 0.f) coef = __fdiv_rn(__fdiv_rn(__fmul_rn(g, __ldg(vis + bk)), S), __fmul_rn((float)HW, r));
        dP[i] = __fmul_rn(coef, __fsub_rn(__ldg(P + i), __ldg(T + i)));
    }
}

// =============================================================================================
// HandSegNet loss (training_handsegnet.py:56-60): mean over rows of softmax_cross_entropy_with_logits for 2 classes, per row as
// TF's SoftmaxXentWithLogits: m = max, e = exp(x - m), s = sum e, loss = sum labels (log s - (x - m)), backprop = e / s - labels.
// =============================================================================================
struct Xent2 { float e0, e1, s, sh0, sh1; };
__device__ __forceinline__ Xent2 xent_row(float2 x) {
    const float m = fmaxf(x.x, x.y);
    Xent2 r;
    r.sh0 = __fsub_rn(x.x, m); r.sh1 = __fsub_rn(x.y, m);
    r.e0 = expf(r.sh0); r.e1 = expf(r.sh1);
    r.s = __fadd_rn(r.e0, r.e1);
    return r;
}

// partial[blk] = sum of the row losses of block blk's row range (thread-strided, then the fixed tree)
__global__ void __launch_bounds__(kRedThreads) xent_partial_kernel(const float2* __restrict__ logits, const float2* __restrict__ labels,
                                                                   float* __restrict__ partial, int64_t rows, int64_t rpb) {
    __shared__ float red[kRedThreads];
    const int64_t r0 = (int64_t)blockIdx.x * rpb, r1 = min(rows, r0 + rpb);
    float s = 0.f;
    for (int64_t r = r0 + threadIdx.x; r < r1; r += kRedThreads) {
        const Xent2 q = xent_row(__ldg(logits + r));
        const float2 l = __ldg(labels + r);
        const float ls = logf(q.s);
        const float row = __fadd_rn(__fmul_rn(l.x, __fsub_rn(ls, q.sh0)), __fmul_rn(l.y, __fsub_rn(ls, q.sh1)));
        s = __fadd_rn(s, row);
    }
    red[threadIdx.x] = s;
    const float tot = block_tree(red);
    if (threadIdx.x == 0) partial[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(kRedThreads) xent_finalize_kernel(const float* __restrict__ partial, int nblk, float* __restrict__ loss,
                                                                    int64_t rows) {
    __shared__ float red[kRedThreads];
    const float tot = block_sum_fixed(partial, nblk, red);
    if (threadIdx.x == 0) *loss = __fdiv_rn(tot, (float)rows);
}

// dlogits = g / N (softmax - labels)
__global__ void xent_grad_kernel(const float2* __restrict__ logits, const float2* __restrict__ labels, const float* __restrict__ grad,
                                 float2* __restrict__ dlogits, int64_t rows) {
    const float scale = __fdiv_rn(grad ? __ldg(grad) : 1.f, (float)rows);
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += (int64_t)gridDim.x * blockDim.x) {
        const Xent2 q = xent_row(__ldg(logits + r));
        const float2 l = __ldg(labels + r);
        dlogits[r] = make_float2(__fmul_rn(scale, __fsub_rn(__fdiv_rn(q.e0, q.s), l.x)), __fmul_rn(scale, __fsub_rn(__fdiv_rn(q.e1, q.s), l.y)));
    }
}

// =============================================================================================
// tf.train.AdamOptimizer (TF 1.3 ApplyAdam, training_ops.cc), one launch for every variable of a network.  state = AdamState: the
// learning rate and the beta powers live on the device, so a captured graph replays the step; the last block to finish (ticket, as
// fc_chain_kernel) advances the powers after every element has used them, as AdamOptimizer._finish does.
// =============================================================================================
struct AdamState { float lr, beta1_power, beta2_power; unsigned int ticket; };
static_assert(sizeof(AdamState) == H3D_ADAM_STATE_WORDS * 4, "AdamState is the header's four-word layout");

constexpr int kAdamChunk = 8192;          // elements per block iteration; a tensor's chunks never straddle into the next tensor
constexpr int kAdamMaxTensors = 1024;
constexpr int kAdamBlocks = 132 * 4;      // one resident wave (5 blocks of 256 threads fit an SM); blocks stride over the chunks

__device__ __forceinline__ void adam_elem(float g, float& m, float& v, float& p, float alpha, float omb1, float omb2, float epsilon) {
    m = __fadd_rn(m, __fmul_rn(__fsub_rn(g, m), omb1));                        // m += (g - m)(1 - beta1)
    v = __fadd_rn(v, __fmul_rn(__fsub_rn(__fmul_rn(g, g), v), omb2));          // v += (g^2 - v)(1 - beta2)
    p = __fsub_rn(p, __fdiv_rn(__fmul_rn(m, alpha), __fadd_rn(__fsqrt_rn(v), epsilon)));   // p -= m alpha / (sqrt(v) + eps)
}

__global__ void __launch_bounds__(kRedThreads) adam_step_kernel(const h3d_adam_tensor* __restrict__ table, int n, AdamState* state,
                                                                float beta1, float beta2, float epsilon) {
    __shared__ int64_t first_chunk[kAdamMaxTensors + 1];
    __shared__ float s_alpha;
    __shared__ bool s_last;
    const int t = threadIdx.x;
    for (int i = t; i < n; i += kRedThreads) first_chunk[i + 1] = (table[i].numel + kAdamChunk - 1) / kAdamChunk;
    __syncthreads();
    if (t == 0) {
        first_chunk[0] = 0;
        for (int i = 1; i <= n; ++i) first_chunk[i] += first_chunk[i - 1];
        const float lr = state->lr, b1p = state->beta1_power, b2p = state->beta2_power;
        // alpha = lr sqrt(1 - beta2^t) / (1 - beta1^t), once per call in fp32, in TF's order
        s_alpha = __fdiv_rn(__fmul_rn(lr, __fsqrt_rn(__fsub_rn(1.f, b2p))), __fsub_rn(1.f, b1p));
    }
    __syncthreads();
    const float alpha = s_alpha, omb1 = __fsub_rn(1.f, beta1), omb2 = __fsub_rn(1.f, beta2);
    const int64_t nchunks = first_chunk[n];
    int ti = 0;
    for (int64_t c = blockIdx.x; c < nchunks; c += gridDim.x) {
        while (first_chunk[ti + 1] <= c) ++ti;     // chunks ascend within a block: the tensor index only moves forward
        const h3d_adam_tensor e = table[ti];
        const int64_t e0 = (c - first_chunk[ti]) * kAdamChunk, e1 = min(e.numel, e0 + kAdamChunk);
        int64_t i = e0 + t;
        // float4 body where all four arrays are 16-byte aligned (chunks start at multiples of 4 elements), scalar tail
        if ((((uintptr_t)e.param | (uintptr_t)e.grad | (uintptr_t)e.m | (uintptr_t)e.v) & 15) == 0) {
            const int64_t e1v = e0 + ((e1 - e0) & ~(int64_t)3);
            for (int64_t j = e0 + 4 * (int64_t)t; j < e1v; j += 4 * kRedThreads) {
                const float4 g = __ldg(reinterpret_cast<const float4*>(e.grad + j));
                float4 m = *reinterpret_cast<const float4*>(e.m + j), v = *reinterpret_cast<const float4*>(e.v + j);
                float4 p = *reinterpret_cast<const float4*>(e.param + j);
                adam_elem(g.x, m.x, v.x, p.x, alpha, omb1, omb2, epsilon);
                adam_elem(g.y, m.y, v.y, p.y, alpha, omb1, omb2, epsilon);
                adam_elem(g.z, m.z, v.z, p.z, alpha, omb1, omb2, epsilon);
                adam_elem(g.w, m.w, v.w, p.w, alpha, omb1, omb2, epsilon);
                *reinterpret_cast<float4*>(e.m + j) = m; *reinterpret_cast<float4*>(e.v + j) = v;
                *reinterpret_cast<float4*>(e.param + j) = p;
            }
            i = e1v + t;
        }
        for (; i < e1; i += kRedThreads) {
            float m = e.m[i], v = e.v[i], p = e.param[i];
            adam_elem(__ldg(e.grad + i), m, v, p, alpha, omb1, omb2, epsilon);
            e.m[i] = m; e.v[i] = v; e.param[i] = p;
        }
    }
    __syncthreads();
    if (t == 0) {
        __threadfence();
        s_last = atomicAdd(&state->ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (s_last && t == 0) {
        __threadfence();
        state->beta1_power = __fmul_rn(state->beta1_power, beta1);
        state->beta2_power = __fmul_rn(state->beta2_power, beta2);
        state->ticket = 0u;                        // ready for the next launch (launches are stream ordered)
    }
}

// mask bit 0: lr, bit 1: beta1_power, bit 2: beta2_power; any write resets the ticket
__global__ void adam_state_set_kernel(AdamState* state, int mask, float lr, float beta1_power, float beta2_power) {
    if (mask & 1) state->lr = lr;
    if (mask & 2) state->beta1_power = beta1_power;
    if (mask & 4) state->beta2_power = beta2_power;
    state->ticket = 0u;
}

int grid_for(int64_t work, int threads) { return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div64(work, threads), 132 * 32)); }

}  // namespace

int64_t resize_grad_scratch_floats(int B, int H, int W, int C, int oh, int ow) {
    return (W != ow && H != oh) ? (int64_t)B * oh * W * C : 0;
}

int launch_resize_bilinear_tf1_grad(const float* dy, float* dx, float* scratch, int B, int H, int W, int C, int oh, int ow, cudaStream_t s,
                                    int* n_launch) {
    *n_launch = 0;
    if (H == oh && W == ow) {   // the forward copies
        H3D_CUDA(cudaMemcpyAsync(dx, dy, (size_t)B * H * W * C * sizeof(float), cudaMemcpyDeviceToDevice, s));
        return H3D_OK;
    }
    const float hscale = (float)H / (float)oh, wscale = (float)W / (float)ow;
    // columns first (dy -> t [B, oh, W, C]); a dimension whose size does not change is the identity and is skipped
    const float* t = dy;
    if (W != ow) {
        float* out = H == oh ? dx : scratch;
        const int64_t total = (int64_t)B * oh * W * C;
        const int blocks = grid_for(total, 256);
        if (C == 21) resize_grad_cols_kernel<21><<<blocks, 256, 0, s>>>(dy, out, (int64_t)B * oh, W, ow, C, wscale);
        else if (C == 2) resize_grad_cols_kernel<2><<<blocks, 256, 0, s>>>(dy, out, (int64_t)B * oh, W, ow, C, wscale);
        else resize_grad_cols_kernel<0><<<blocks, 256, 0, s>>>(dy, out, (int64_t)B * oh, W, ow, C, wscale);
        H3D_CHECK_LAUNCH();
        ++*n_launch;
        t = out;
    }
    if (H != oh) {
        resize_grad_rows_kernel<<<grid_for((int64_t)B * H * W * C, 256), 256, 0, s>>>(t, dx, B, H, oh, (int64_t)W * C, hscale);
        H3D_CHECK_LAUNCH();
        ++*n_launch;
    }
    return H3D_OK;
}

// Chunks per image of the score-map reduction: about two blocks per SM over the batch, at least 256 pixels each (shape-only policy)
static int scoremap_chunks(int B, int HW) { return std::max(1, std::min(ceil_div(HW, 256), ceil_div(264, B))); }

int64_t scoremap_loss_scratch_floats(int B, int H, int W) { return (int64_t)B * scoremap_chunks(B, H * W) * kSmK; }

int launch_scoremap_loss(const float* P, const float* T, const float* vis, float* scratch, int B, int H, int W, float* loss, float* rms,
                         cudaStream_t s) {
    const int HW = H * W, nchunk = scoremap_chunks(B, HW), ppc = ceil_div(HW, nchunk);
    scoremap_sq_partial_kernel<<<dim3(nchunk, B), kSmThreads, 0, s>>>(P, T, scratch, HW, ppc, nchunk);
    H3D_CHECK_LAUNCH();
    scoremap_loss_finalize_kernel<<<1, kRedThreads, 0, s>>>(scratch, vis, rms, loss, B * kSmK, HW, nchunk);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

int launch_scoremap_loss_grad(const float* P, const float* T, const float* vis, const float* rms, const float* grad, float* dP, int B,
                              int H, int W, cudaStream_t s) {
    const int64_t total = (int64_t)B * H * W * kSmK;
    scoremap_loss_grad_kernel<<<grid_for(total, kRedThreads * 8), kRedThreads, 0, s>>>(P, T, vis, rms, grad, dP, B * kSmK, H * W);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

// Blocks of the cross-entropy reduction: at most 1024, at least 2048 rows each (shape-only policy)
static int xent_blocks(int64_t rows, int64_t* rpb) {
    const int64_t nblk = std::max<int64_t>(1, std::min<int64_t>(ceil_div64(rows, 2048), 1024));
    *rpb = ceil_div64(rows, nblk);
    return (int)ceil_div64(rows, *rpb);
}

int64_t softmax_xent_scratch_floats(int64_t rows) { int64_t rpb; return xent_blocks(rows, &rpb); }

int launch_softmax_xent(const float* logits, const float* labels, float* scratch, int64_t rows, float* loss, cudaStream_t s) {
    int64_t rpb = 0;
    const int nblk = xent_blocks(rows, &rpb);
    xent_partial_kernel<<<nblk, kRedThreads, 0, s>>>((const float2*)logits, (const float2*)labels, scratch, rows, rpb);
    H3D_CHECK_LAUNCH();
    xent_finalize_kernel<<<1, kRedThreads, 0, s>>>(scratch, nblk, loss, rows);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

int launch_softmax_xent_grad(const float* logits, const float* labels, const float* grad, float* dlogits, int64_t rows, cudaStream_t s) {
    xent_grad_kernel<<<grid_for(rows, 256 * 4), 256, 0, s>>>((const float2*)logits, (const float2*)labels, grad, (float2*)dlogits, rows);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

int launch_adam_step(const h3d_adam_tensor* table, int n, float* state, float beta1, float beta2, float epsilon, cudaStream_t s) {
    H3D_REQUIRE(n >= 1 && n <= kAdamMaxTensors, "h3d_adam_step: 1 to %d tensors per call", kAdamMaxTensors);
    adam_step_kernel<<<kAdamBlocks, kRedThreads, 0, s>>>(table, n, (AdamState*)state, beta1, beta2, epsilon);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

int launch_adam_state_set(float* state, int mask, float lr, float beta1_power, float beta2_power, cudaStream_t s) {
    adam_state_set_kernel<<<1, 1, 0, s>>>((AdamState*)state, mask, lr, beta1_power, beta2_power);
    H3D_CHECK_LAUNCH();
    return H3D_OK;
}

}  // namespace h3d

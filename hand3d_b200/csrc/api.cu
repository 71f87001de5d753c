// C ABI (include/hand3d_b200.h): context, weight loading / packing, workspace layout, the fixed layer
// schedules of HandSegNet / PoseNet2D / PosePrior / ViewpointNet and the full pipeline.
#include <cstdarg>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "common.cuh"
#include "split_fmt.cuh"

namespace h3d {

// ------------------------------------------------------------------------------------------ errors
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
int cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
    set_error("CUDA error %d (%s) at %s:%d: %s", (int)e, cudaGetErrorString(e), file, line, what);
    if (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver) return H3D_ENODEVICE;
    return H3D_ECUDA;
}

// ------------------------------------------------------------------------------------------ layer tables
struct LayerSpec { const char* name; int k, stride, cin, cout, leaky; };

static const LayerSpec kHandSeg[] = {
    {"conv1_1", 3, 1, 3, 64, 1},    {"conv1_2", 3, 1, 64, 64, 1},   {"conv2_1", 3, 1, 64, 128, 1},  {"conv2_2", 3, 1, 128, 128, 1},
    {"conv3_1", 3, 1, 128, 256, 1}, {"conv3_2", 3, 1, 256, 256, 1}, {"conv3_3", 3, 1, 256, 256, 1}, {"conv3_4", 3, 1, 256, 256, 1},
    {"conv4_1", 3, 1, 256, 512, 1}, {"conv4_2", 3, 1, 512, 512, 1}, {"conv4_3", 3, 1, 512, 512, 1}, {"conv4_4", 3, 1, 512, 512, 1},
    {"conv5_1", 3, 1, 512, 512, 1}, {"conv5_2", 3, 1, 512, 128, 1}, {"conv6_1", 1, 1, 128, 512, 1}, {"conv6_2", 1, 1, 512, 2, 0}};
static const LayerSpec kPoseTrunk[] = {
    {"conv1_1", 3, 1, 3, 64, 1},    {"conv1_2", 3, 1, 64, 64, 1},   {"conv2_1", 3, 1, 64, 128, 1},  {"conv2_2", 3, 1, 128, 128, 1},
    {"conv3_1", 3, 1, 128, 256, 1}, {"conv3_2", 3, 1, 256, 256, 1}, {"conv3_3", 3, 1, 256, 256, 1}, {"conv3_4", 3, 1, 256, 256, 1},
    {"conv4_1", 3, 1, 256, 512, 1}, {"conv4_2", 3, 1, 512, 512, 1}, {"conv4_3", 3, 1, 512, 256, 1}, {"conv4_4", 3, 1, 256, 256, 1},
    {"conv4_5", 3, 1, 256, 256, 1}, {"conv4_6", 3, 1, 256, 256, 1}, {"conv4_7", 3, 1, 256, 128, 1}};
static const LayerSpec kPosePrior[] = {{"conv_pose_0_1", 3, 1, 21, 32, 1},  {"conv_pose_0_2", 3, 2, 32, 32, 1},
                                       {"conv_pose_1_1", 3, 1, 32, 64, 1},  {"conv_pose_1_2", 3, 2, 64, 64, 1},
                                       {"conv_pose_2_1", 3, 1, 64, 128, 1}, {"conv_pose_2_2", 3, 2, 128, 128, 1}};
static const LayerSpec kViewpoint[] = {{"conv_vp_0_1", 3, 1, 21, 64, 1},   {"conv_vp_0_2", 3, 2, 64, 64, 1},
                                       {"conv_vp_1_1", 3, 1, 64, 128, 1},  {"conv_vp_1_2", 3, 2, 128, 128, 1},
                                       {"conv_vp_2_1", 3, 1, 128, 256, 1}, {"conv_vp_2_2", 3, 2, 256, 256, 1}};

struct VarShape { int nd; int64_t s[4]; };
static std::map<std::string, VarShape> build_known_vars() {
    std::map<std::string, VarShape> m;
    auto conv = [&](const std::string& scope, const LayerSpec& l) {
        m[scope + "/" + l.name + "/weights"] = {4, {l.k, l.k, l.cin, l.cout}};
        m[scope + "/" + l.name + "/biases"] = {1, {l.cout, 0, 0, 0}};
    };
    auto fc = [&](const std::string& scope, const char* n, int in, int out) {
        m[scope + "/" + n + "/weights"] = {2, {in, out, 0, 0}};
        m[scope + "/" + n + "/biases"] = {1, {out, 0, 0, 0}};
    };
    for (auto& l : kHandSeg) conv("HandSegNet", l);
    for (auto& l : kPoseTrunk) conv("PoseNet2D", l);
    conv("PoseNet2D", {"conv5_1", 1, 1, 128, 512, 1});
    conv("PoseNet2D", {"conv5_2", 1, 1, 512, 21, 0});
    for (int u = 6; u <= 7; ++u) {
        char nm[16];
        for (int i = 1; i <= 7; ++i) {
            snprintf(nm, sizeof(nm), "conv%d_%d", u, i);
            const int k = i <= 5 ? 7 : 1, cin = i == 1 ? 149 : 128, cout = i == 7 ? 21 : 128;
            m[std::string("PoseNet2D/") + nm + "/weights"] = {4, {k, k, cin, cout}};
            m[std::string("PoseNet2D/") + nm + "/biases"] = {1, {cout, 0, 0, 0}};
        }
    }
    for (auto& l : kPosePrior) conv("PosePrior", l);
    fc("PosePrior", "fc_rel0", 2050, 512); fc("PosePrior", "fc_rel1", 512, 512); fc("PosePrior", "fc_xyz", 512, 63);
    fc("PosePrior", "fc_bottleneck", 512, 30);
    for (auto& l : kViewpoint) conv("ViewpointNet", l);
    fc("ViewpointNet", "fc_vp0", 4098, 256); fc("ViewpointNet", "fc_vp1", 256, 128);
    fc("ViewpointNet", "fc_vp_ux", 128, 1); fc("ViewpointNet", "fc_vp_uy", 128, 1); fc("ViewpointNet", "fc_vp_uz", 128, 1);
    return m;
}
static const std::map<std::string, VarShape>& known_vars() {
    static const std::map<std::string, VarShape> m = build_known_vars();
    return m;
}

// ------------------------------------------------------------------------------------------ context
struct HostTensor { std::vector<float> data; std::vector<int64_t> shape; };
// w_scale: fp16 planes with passes 1 / 3, the per-channel shift factors 2^-s (split_fmt.cuh), stored after the padded bias
struct PackedW { Split w; float* bias = nullptr; float* w_scale = nullptr; int Cin_pad = 0, Cout_pad = 0; float corr_scale = 0.f; };

struct Arena {   // bump allocator over the caller-owned workspace (base == nullptr -> size query)
    char* base = nullptr; int64_t off = 0;
    template <typename T> T* alloc(int64_t n) {
        off = align_up(off, 1024);
        T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off += n * (int64_t)sizeof(T);
        return p;
    }
};

struct Ext {   // pointers that change per call (everything else is baked into the plan)
    const float* in = nullptr;
    float* out = nullptr;
    float* out2 = nullptr;
    float* out3 = nullptr;
    const float* hand_side = nullptr;
};
using StepFn = std::function<int(const Ext&, cudaStream_t)>;

enum StepKind { KIND_TC = 0, KIND_DIRECT = 1, KIND_FC = 2, KIND_OTHER = 3, KIND_COUNT = 4 };

struct StagePlan {
    std::vector<StepFn> steps;
    std::vector<int> launches;          // kernels per step
    std::vector<int> kinds;             // StepKind per step (profiling)
    std::vector<int64_t> step_flops;    // algorithmic FLOPs per step
    std::vector<TcConvPlan*> tc;
    std::vector<FcChainPlan*> fc;
    std::vector<int> lane;              // per step: 0 = caller's stream, 1 = the context's side stream (independent branch)
    std::vector<char> join_before;      // per step: wait for the side stream before this step
    int cur_lane = 0;                   // lane given to steps as they are appended (see seal())
    int B = 0, H = 0, W = 0, variant = -1;
    int64_t flops = 0;
    // layer chains (per chained launch one ticket word + B per-image completion counters, zeroed by the plan's first step;
    // chain_prev = the chained launch appended last, iff it is the plan's most recent step): only for plans that
    // tc_conv_plan_chainable() accepts, none in the sm_90a build
    int* sync = nullptr;
    int sync_slots = 0;
    TcConvPlan* chain_prev = nullptr;
    size_t chain_prev_step = 0;
    int* chain_prev_sig = nullptr;
    ~StagePlan() {
        for (auto* p : tc) tc_conv_plan_destroy(p);
        for (auto* p : fc) fc_chain_plan_destroy(p);
        if (sync) cudaFree(sync);
    }
    // label every step appended since the last call with the current lane
    void seal(bool join = false) {
        const size_t first = lane.size();
        while (lane.size() < steps.size()) { lane.push_back(cur_lane); join_before.push_back(0); }
        if (join && first < steps.size()) join_before[first] = 1;
    }
};

}  // namespace h3d

using namespace h3d;

struct h3d_ctx {
    int device = 0;
    int precision = H3D_PREC_BF16X3;
    int64_t launches = 0;
    std::map<std::string, HostTensor> host_w;
    std::map<std::string, float*> dev_w;          // raw fp32 copies (HWIO / [in,out] / [C]) for the CUDA-core kernels
    std::map<std::string, PackedW> packed;        // key = name|half|perm
    float* vp_head_w = nullptr; float* vp_head_b = nullptr;   // fused fc_vp_ux/uy/uz [128,3]
    char* ws = nullptr; int64_t ws_bytes = 0;
    std::unique_ptr<StagePlan> seg, pose, lift;
    // persistent buffers inside the workspace (laid out by layout())
    struct Layout {
        int B = 0, H = 0, W = 0;
        float *hand_scoremap, *image_crop, *kp_scoremap, *center, *scale, *crop_size, *coord3d;
        int32_t* kp_uv;
        void *seg_scratch, *argmax_scratch;
        float *seg_low, *s[3];
        int64_t seg_off, pose_off, lift_off, total;
    } lay;
    void drop_plans() { seg.reset(); pose.reset(); lift.reset(); }
    // independent branches (PosePrior || ViewpointNet, x8 up-sampling || lifting) run on two private streams that fork from
    // and join back into the caller's stream with events (capturable into a CUDA graph)
    cudaStream_t side = nullptr, side2 = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr, ev_fork2 = nullptr, ev_join2 = nullptr;
    // Device-visible error word in pinned host memory: a bounded barrier wait that times out stores its code here (system-scope
    // atomic) before trapping, and the gather kernel stores 100 + peer when a peer never signals.  Readable by the host even
    // after the trap has poisoned the CUDA context (h3d_check_errors).
    int* err_flag = nullptr;
    unsigned int* fc_counter = nullptr;      // ticket of the FC-chain kernel ("last cluster applies the rotation epilogue"), zero between launches
    // Operator entry points borrow scratch from here instead of allocating per call: grown geometrically on demand, old blocks
    // are retired (not freed) until h3d_destroy, so no call ever synchronises or frees.
    char* op_scratch = nullptr; int64_t op_scratch_bytes = 0;
    std::vector<void*> retired;
    // optional per-kernel-class timing (CUDA events on the launch stream around every plan step)
    bool profiling = false;
    struct ProfRec { cudaEvent_t a, b; int kind; int64_t flops; };
    std::vector<ProfRec> prof;
};

namespace h3d {

static bool is_tc(int precision) { return precision != H3D_PREC_FP32_FFMA; }
// 1 = single 16-bit pass, 3 = hi/lo 16-bit planes (3 MMA passes), 4 = fp16 plane + e4m3 residual / coarse planes (1 fp16 + 2 fp8 passes)
static int passes_of(int precision) {
    if (precision == H3D_PREC_FP16_F8C) return 4;
    return (precision == H3D_PREC_BF16X3 || precision == H3D_PREC_FP16X3) ? 3 : 1;
}
static Half16 half_of(int precision) {
    return (precision == H3D_PREC_FP16X3 || precision == H3D_PREC_FP16 || precision == H3D_PREC_FP16_F8C) ? Half16::FP16 : Half16::BF16;
}

static uint16_t host_h16(float v, Half16 t) {
    if (t == Half16::FP16) { __half h = __float2half_rn(v); uint16_t b; memcpy(&b, &h, 2); return b; }
    __nv_bfloat16 h = __float2bfloat16_rn(v); uint16_t b; memcpy(&b, &h, 2); return b;
}
static float host_f32(uint16_t b, Half16 t) {
    if (t == Half16::FP16) { __half h; memcpy(&h, &b, 2); return __half2float(h); }
    uint32_t u = (uint32_t)b << 16; float f; memcpy(&f, &u, 4); return f;
}

// Pack HWIO fp32 -> K-major [Cout_pad][kh][kw][Cin_pad] hi/lo planes.  perm[j] = source input channel of
// packed channel j (or -1 for zero padding); empty perm = identity.  fp16 planes (passes 1 / 3) carry the per-channel weight shift
// of split_fmt.cuh; its factors 2^-s follow the padded bias in the same allocation ([bias | w_scale], 2 Cout_pad floats).
static int pack_conv_weights(const float* w, const float* bias, int k, int Cin, int Cout, int Cin_pad, int Cout_pad,
                             const std::vector<int>& perm, Half16 t, int passes, PackedW* out) {
    const int64_t Ktot = (int64_t)k * k * Cin_pad;
    const bool want_lo = passes == 3, f8c = passes == 4, shifted = t == Half16::FP16 && !f8c;
    std::vector<uint16_t> hi((size_t)Cout_pad * Ktot, 0), lo;
    std::vector<uint8_t> h8, l8;
    if (want_lo) lo.assign((size_t)Cout_pad * Ktot, 0);
    int b = 0;
    if (f8c) {
        // e4m3 planes: wh8 = e4m3(w 2^b), wl8 = e4m3((w - fp16(w)) 2^(12+b)); b puts max|w| just below the e4m3 maximum (448).
        // Paired with the activation planes (l8 = residual 2^10, h8 = x 2^-2) both fp8 products carry 2^(10+b).
        float mx = 0.f;
        for (int64_t i = 0; i < (int64_t)k * k * Cin * Cout; ++i) mx = std::max(mx, std::fabs(w[i]));
        b = mx > 0.f ? (int)std::floor(std::log2(240.0f / mx)) : 0;
        b = std::max(-20, std::min(20, b));
        h8.assign((size_t)Cout_pad * Ktot, 0); l8.assign((size_t)Cout_pad * Ktot, 0);
        out->corr_scale = std::ldexp(1.0f, -(kF8XLoShift + b));
    }
    std::vector<int> sh((size_t)Cout_pad, 0);
    if (shifted)
        for (int co = 0; co < Cout; ++co) {
            float mx = 0.f;
            for (int64_t r = 0; r < (int64_t)k * k * Cin; ++r) mx = std::max(mx, std::fabs(w[r * Cout + co]));
            sh[co] = fp16_w_shift(mx);
        }
    for (int co = 0; co < Cout; ++co)
        for (int tap = 0; tap < k * k; ++tap)
            for (int cj = 0; cj < Cin_pad; ++cj) {
                const int ci = perm.empty() ? (cj < Cin ? cj : -1) : perm[cj];
                if (ci < 0) continue;
                const float v = w[((int64_t)tap * Cin + ci) * Cout + co];
                const int64_t idx = (int64_t)co * Ktot + (int64_t)tap * Cin_pad + cj;
                if (f8c) {   // all three planes pre-scaled so that every operand product carries 2^(10+b) (see split_fmt.cuh)
                    const uint16_t h = host_h16(std::ldexp(v, kF8XMainShift + b), t);
                    hi[idx] = h;
                    h8[idx] = f32_to_e4m3(std::ldexp(v, b));
                    l8[idx] = f32_to_e4m3(std::ldexp(v - std::ldexp(host_f32(h, t), -(kF8XMainShift + b)), 12 + b));
                    continue;
                }
                const float vs = std::ldexp(v, sh[co]);
                const uint16_t h = host_h16(vs, t);
                hi[idx] = h;
                if (want_lo) lo[idx] = host_h16(vs - host_f32(h, t), t);
            }
    std::vector<float> bv((size_t)Cout_pad, 0.f);
    for (int co = 0; co < Cout; ++co) bv[co] = bias[co];
    if (shifted)
        for (int co = 0; co < Cout_pad; ++co) bv.push_back(std::ldexp(1.0f, -sh[co]));
    H3D_CUDA(cudaMalloc(&out->w.hi, hi.size() * 2));
    H3D_CUDA(cudaMemcpy(out->w.hi, hi.data(), hi.size() * 2, cudaMemcpyHostToDevice));
    if (want_lo) {
        H3D_CUDA(cudaMalloc(&out->w.lo, lo.size() * 2));
        H3D_CUDA(cudaMemcpy(out->w.lo, lo.data(), lo.size() * 2, cudaMemcpyHostToDevice));
    }
    if (f8c) {
        H3D_CUDA(cudaMalloc(&out->w.h8, h8.size())); H3D_CUDA(cudaMalloc(&out->w.l8, l8.size()));
        H3D_CUDA(cudaMemcpy(out->w.h8, h8.data(), h8.size(), cudaMemcpyHostToDevice));
        H3D_CUDA(cudaMemcpy(out->w.l8, l8.data(), l8.size(), cudaMemcpyHostToDevice));
    }
    H3D_CUDA(cudaMalloc(&out->bias, bv.size() * 4));
    H3D_CUDA(cudaMemcpy(out->bias, bv.data(), bv.size() * 4, cudaMemcpyHostToDevice));
    if (shifted) out->w_scale = out->bias + Cout_pad;
    out->Cin_pad = Cin_pad; out->Cout_pad = Cout_pad;
    return H3D_OK;
}

static void free_packed(PackedW& p) {
    if (p.w.hi) cudaFree(p.w.hi);
    if (p.w.lo) cudaFree(p.w.lo);
    if (p.w.l8) cudaFree(p.w.l8);
    if (p.w.h8) cudaFree(p.w.h8);
    if (p.bias) cudaFree(p.bias);
    p = PackedW();
}

// RAII: make ctx's device current for the duration of an entry point and restore the caller's device afterwards (one process may
// hold contexts on several GPUs; torch keeps its own notion of the current device).
struct DeviceGuard {
    int prev = -1; bool switched = false;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) == cudaSuccess && prev != dev) switched = cudaSetDevice(dev) == cudaSuccess;
    }
    ~DeviceGuard() { if (switched) cudaSetDevice(prev); }
};

static int op_scratch(h3d_ctx* ctx, int64_t bytes, char** out) {
    if (ctx->op_scratch_bytes < bytes) {
        const int64_t want = std::max<int64_t>(align_up(bytes, 1 << 20), 2 * ctx->op_scratch_bytes);
        char* p = nullptr;
        H3D_CUDA(cudaMalloc(&p, (size_t)want));
        if (ctx->op_scratch) ctx->retired.push_back(ctx->op_scratch);   // in-flight kernels may still use it
        ctx->op_scratch = p; ctx->op_scratch_bytes = want;
    }
    *out = ctx->op_scratch;
    return H3D_OK;
}

static int get_packed(h3d_ctx* ctx, const std::string& scope, const LayerSpec& l, int Cin_pad, const std::vector<int>& perm,
                      const PackedW** out, int force_passes = 0) {
    const Half16 t = half_of(ctx->precision);
    const int passes = force_passes ? force_passes : passes_of(ctx->precision);
    const std::string key = scope + "/" + l.name + (t == Half16::FP16 ? "|h" : "|b") + std::to_string(passes);
    auto it = ctx->packed.find(key);
    if (it == ctx->packed.end()) {
        auto wi = ctx->host_w.find(scope + "/" + l.name + "/weights"), bi = ctx->host_w.find(scope + "/" + l.name + "/biases");
        if (wi == ctx->host_w.end() || bi == ctx->host_w.end()) { set_error("weights for %s/%s not loaded", scope.c_str(), l.name); return H3D_EWEIGHTS; }
        PackedW p;
        int rc = pack_conv_weights(wi->second.data.data(), bi->second.data.data(), l.k, l.cin, l.cout, Cin_pad, (int)align_up(l.cout, 64), perm, t, passes, &p);
        if (rc) return rc;
        it = ctx->packed.emplace(key, p).first;
    }
    *out = &it->second;
    return H3D_OK;
}

static int dev_weight(h3d_ctx* ctx, const std::string& name, const float** out) {
    auto it = ctx->dev_w.find(name);
    if (it == ctx->dev_w.end()) { set_error("weights %s not loaded", name.c_str()); return H3D_EWEIGHTS; }
    *out = it->second;
    return H3D_OK;
}

// ------------------------------------------------------------------------------------------ workspace layout
static int64_t slot_elems_seg(int B, int H, int W) { return (int64_t)B * H * W * 64; }

// FC split-K scratch of one lifting branch on the CUDA-core path: the maximum of fc_scratch_floats over the stage's FC shapes.
// fc_ksplit chooses each layer's split count from its tile count, so the widest layer is not always the one that needs the most
// (fc_vp0, 4098 -> 256, needs more than fc_rel0, 2050 -> 512, at B = 33 ... 64 for example).
static int64_t lift_fc_scratch_floats(int B) {
    static const int shapes[][2] = {{2050, 512}, {512, 512}, {512, 30}, {512, 63}, {30, 63},   // PosePrior, incl. the bottleneck
                                    {4098, 256}, {256, 128}, {128, 3}};                         // ViewpointNet, fused ux | uy | uz heads
    int64_t m = 0;
    for (const auto& sh : shapes) m = std::max(m, fc_scratch_floats(B, sh[0], sh[1]));
    return m;
}

static void layout(h3d_ctx::Layout& L, char* base, int B, int H, int W) {
    Arena a; a.base = base;
    L.B = B; L.H = H; L.W = W;
    L.hand_scoremap = a.alloc<float>((int64_t)B * H * W * 2);
    L.image_crop = a.alloc<float>((int64_t)B * 256 * 256 * 3);
    L.kp_scoremap = a.alloc<float>((int64_t)B * 256 * 256 * 21);
    L.center = a.alloc<float>(B * 2); L.scale = a.alloc<float>(B); L.crop_size = a.alloc<float>(B);
    L.coord3d = a.alloc<float>(B * 63);
    L.kp_uv = a.alloc<int32_t>(B * 42);
    L.seg_scratch = a.alloc<char>(seg_scratch_bytes(B, H, W));
    L.argmax_scratch = a.alloc<char>(argmax_scratch_bytes(B, 21));
    L.seg_low = a.alloc<float>((int64_t)B * (H / 8) * (W / 8) * 2);
    const int Hc = std::max(H, 256), Wc = std::max(W, 256);   // PoseNet may also be called stand-alone on HxW crops
    for (int i = 0; i < 3; ++i) L.s[i] = a.alloc<float>((int64_t)B * (Hc / 8) * (Wc / 8) * 21);
    a.off = align_up(a.off, 1024); L.seg_off = a.off;
    a.off += 2 * align_up(slot_elems_seg(B, H, W) * 4, 1024) + 4096;
    a.off = align_up(a.off, 1024); L.pose_off = a.off;
    a.off += 2 * align_up((int64_t)B * Hc * Wc * 64 * 4, 1024) + 2 * align_up((int64_t)B * (Hc / 8) * (Wc / 8) * 192 * 4, 1024) +
             align_up((int64_t)B * (Hc / 8) * (Wc / 8) * 512 * 4, 1024) + 8192;
    a.off = align_up(a.off, 1024); L.lift_off = a.off;
    // lifting: input planes + two ping-pong slots per branch (PosePrior, ViewpointNet), FC buffers and scratch per branch
    a.off += 5 * align_up((int64_t)B * 32 * 32 * 64 * 4, 1024) + 2 * 5 * align_up((int64_t)B * 4100 * 4, 1024) +
             2 * align_up(lift_fc_scratch_floats(B) * 4, 1024) + 2 * align_up(kConvSplitKScratchFloats * 4, 1024) + 65536;
    L.total = align_up(a.off, 1024);
}

static int ensure_layout(h3d_ctx* ctx, int B, int H, int W) {
    h3d_ctx::Layout probe;
    layout(probe, nullptr, B, H, W);
    if (!ctx->ws || ctx->ws_bytes < probe.total) {
        set_error("workspace too small: need %lld bytes for B=%d H=%d W=%d, have %lld (call h3d_workspace_bytes / h3d_set_workspace)",
                  (long long)probe.total, B, H, W, (long long)ctx->ws_bytes);
        return H3D_EWORKSPACE;
    }
    if (ctx->lay.B != B || ctx->lay.H != H || ctx->lay.W != W || ctx->lay.hand_scoremap != (float*)ctx->ws) {
        ctx->drop_plans();
        layout(ctx->lay, ctx->ws, B, H, W);
    }
    return H3D_OK;
}

// A stage call fits the current layout when its batch and spatial sizes are covered by what layout(B,H,W) reserved
// (HandSegNet slots for HxW, PoseNet slots for max(H,256) x max(W,256), lifting for B); otherwise the layout grows to
// the element-wise maximum (which needs a workspace sized for it).
static int ensure_layout_covers(h3d_ctx* ctx, int B, int segH, int segW, int poseH, int poseW) {
    const h3d_ctx::Layout& L = ctx->lay;
    const bool have = ctx->ws && L.hand_scoremap == (float*)ctx->ws && L.B > 0;
    if (have && B <= L.B && segH <= L.H && segW <= L.W && poseH <= std::max(L.H, 256) && poseW <= std::max(L.W, 256)) return H3D_OK;
    int nB = B, nH = std::max(segH, 8), nW = std::max(segW, 8);
    if (poseH > 256) nH = std::max(nH, poseH);
    if (poseW > 256) nW = std::max(nW, poseW);
    if (have) { nB = std::max(nB, L.B); nH = std::max(nH, L.H); nW = std::max(nW, L.W); }
    return ensure_layout(ctx, nB, nH, nW);
}

// ------------------------------------------------------------------------------------------ step builders
struct Act {   // an activation tensor living in the workspace
    float* f = nullptr;   // fp32 view
    Split s;              // split view (tensor-core modes)
    int C = 0;            // channel stride
};
// planes of one activation tensor inside a slot of 4 bytes / element: passes 3 -> [hi 2B | lo 2B]; 4 -> [fp16 2B | l8 1B | h8 1B]
static Act slot_view(char* p, int64_t elems, int C, bool split, int passes) {
    Act a; a.C = C;
    if (!split) { a.f = (float*)p; return a; }
    a.s.hi = (uint16_t*)p;
    if (passes == 3) a.s.lo = (uint16_t*)(p + align_up(elems * 2, 1024));
    if (passes == 4) {
        a.s.l8 = (uint8_t*)(p + align_up(elems * 2, 1024));
        a.s.h8 = a.s.l8 + align_up(elems, 1024);
    }
    return a;
}

static void tag(StagePlan* pl, int kind, int64_t flops) {
    while (pl->kinds.size() + 1 < pl->launches.size()) { pl->kinds.push_back(KIND_OTHER); pl->step_flops.push_back(0); }
    pl->kinds.push_back(kind); pl->step_flops.push_back(flops);
}

static int add_direct(h3d_ctx* ctx, StagePlan* pl, const std::string& scope, const LayerSpec& l, int B, int H, int W,
                      const float* x /*null -> Ext.in*/, int Cin_total, int cin_off, float* y, int Cout_total, int cout_off,
                      Split ys, int Cs_total, int cs_off, float* splitk_scratch = nullptr) {
    const float *w, *b;
    int rc;
    if ((rc = dev_weight(ctx, scope + "/" + l.name + "/weights", &w))) return rc;
    if ((rc = dev_weight(ctx, scope + "/" + l.name + "/biases", &b))) return rc;
    DirectConvArgs a;
    a.x = x; a.Cin_total = Cin_total; a.cin_off = cin_off; a.w = w; a.bias = b; a.y = y; a.Cout_total = Cout_total; a.cout_off = cout_off;
    a.ys = ys; a.Cs_total = Cs_total; a.cs_off = cs_off; a.half = half_of(ctx->precision);
    a.B = B; a.H = H; a.W = W; a.Cin = l.cin; a.Cout = l.cout; a.k = l.k; a.stride = l.stride; a.leaky = l.leaky;
    a.splitk_scratch = splitk_scratch; a.splitk_scratch_floats = splitk_scratch ? kConvSplitKScratchFloats : 0;
    a.err_flag = ctx->err_flag;
    pl->steps.push_back([a](const Ext& e, cudaStream_t s) {
        DirectConvArgs aa = a;
        if (!aa.x) aa.x = e.in;
        return launch_conv_direct(aa, s);
    });
    pl->launches.push_back(conv_direct_num_launches(a));
    const int64_t fl = 2ll * B * ceil_div(H, l.stride) * ceil_div(W, l.stride) * l.k * l.k * l.cin * l.cout;
    pl->flops += fl;
    tag(pl, KIND_DIRECT, fl);
    return H3D_OK;
}

constexpr int kMaxChainSlots = 96;

// First step of a stage plan that chains layers: zero the ticket words and completion counters (one memset node per stage call)
static int begin_chain_sync(StagePlan* pl, int B) {
    if (!tc_tuning().chain) return H3D_OK;
    const size_t bytes = (size_t)kMaxChainSlots * (B + 1) * sizeof(int);
    H3D_CUDA(cudaMalloc(&pl->sync, bytes));   // plan build time, never on a launch path
    int* sync = pl->sync;
    pl->steps.push_back([sync, bytes](const Ext&, cudaStream_t s) { H3D_CUDA(cudaMemsetAsync(sync, 0, bytes, s)); return H3D_OK; });
    pl->launches.push_back(0);
    return H3D_OK;
}

static int add_tc(h3d_ctx* ctx, StagePlan* pl, const std::string& scope, const LayerSpec& l, int B, int H, int W, Split x,
                  int Cin_total, int Cin_pad, const std::vector<int>& perm, Split y, int Cy_total, int cy_off, float* yf,
                  int Cyf_total, int cyf_off, int pool = 0, int force_passes = 0, bool chain = false, const LayerSpec* first = nullptr) {
    const PackedW* pw;
    int rc = get_packed(ctx, scope, l, Cin_pad, perm, &pw, force_passes);
    if (rc) return rc;
    TcConvDesc d;
    d.x = x; d.Cin_total = Cin_total; d.Cin_pad = Cin_pad; d.w = pw->w; d.bias = pw->bias; d.w_scale = pw->w_scale; d.Cout = l.cout;
    d.Cout_pad = pw->Cout_pad;
    d.y = y; d.Cy_total = Cy_total; d.cy_off = cy_off; d.yf = yf; d.Cyf_total = Cyf_total; d.cyf_off = cyf_off;
    d.B = B; d.H = H; d.W = W; d.k = l.k; d.leaky = l.leaky; d.passes = force_passes ? force_passes : passes_of(ctx->precision);
    d.half = half_of(ctx->precision);
    d.corr_scale = pw->corr_scale;
    d.pool = pool;
    d.err_flag = ctx->err_flag;
    if (first) {   // conv1_1 (fp32 image -> 64 channels) is computed inside this layer's kernel; its input comes from Ext.in at launch
        if ((rc = dev_weight(ctx, scope + "/" + first->name + "/weights", &d.c1_w))) return rc;
        if ((rc = dev_weight(ctx, scope + "/" + first->name + "/biases", &d.c1_bias))) return rc;
        d.c1_leaky = first->leaky;
    }
    TcConvPlan* tp = tc_conv_plan_create(d);
    if (!tp) return H3D_ECUDA;
    pl->tc.push_back(tp);
    if (chain && pl->sync && tc_conv_plan_chainable(tp) && pl->sync_slots < kMaxChainSlots) {
        int* words = pl->sync + (size_t)pl->sync_slots++ * (B + 1);   // [ticket | completion counter per image]
        const int* dep = nullptr; int target = 0;
        if (tc_tuning().chain == 1 && pl->chain_prev && pl->chain_prev_step + 1 == pl->steps.size()) {
            // the previous step is a chained launch: depend on it per image iff it produces ALL of this layer's input planes
            const TcConvDesc& pd = tc_conv_plan_desc(pl->chain_prev);
            const int ph = pd.pool ? pd.H / 2 : pd.H, pw = pd.pool ? pd.W / 2 : pd.W;
            if (pd.y.hi == x.hi && pd.y.lo == x.lo && pd.y.l8 == x.l8 && pd.cy_off == 0 && pd.Cy_total == Cin_total && pd.Cout_pad == Cin_pad &&
                pd.B == B && ph == H && pw == W) {
                dep = pl->chain_prev_sig; target = tc_conv_plan_signal_target(pl->chain_prev);
            }
        }
        tc_conv_plan_set_chain(tp, words, dep, target, words + 1);
        pl->chain_prev = tp; pl->chain_prev_step = pl->steps.size(); pl->chain_prev_sig = words + 1;
    }
    if (first) pl->steps.push_back([tp](const Ext& e, cudaStream_t s) { return tc_conv_launch_image(tp, e.in, s); });
    else pl->steps.push_back([tp](const Ext&, cudaStream_t s) { return tc_conv_launch(tp, s); });
    pl->launches.push_back(1);
    const int64_t fl = 2ll * B * H * W * l.k * l.k * l.cin * l.cout / (pool == 2 ? 4 : 1) +
                       (first ? 2ll * B * H * W * first->k * first->k * first->cin * first->cout : 0);
    pl->flops += fl;
    tag(pl, KIND_TC, fl);
    return H3D_OK;
}

// VGG-style trunk shared by HandSegNet and PoseNet2D: conv layers [0, n) of `layers` with 2x2 pools after
// conv1_2 / conv2_2 / conv3_4; ping-pongs between two workspace slots.  Returns the final activation.
static int build_trunk(h3d_ctx* ctx, StagePlan* pl, const std::string& scope, const LayerSpec* layers, int n, int B, int H, int W,
                       char* slot0, char* slot1, int64_t slot_elems, Act* last, int* Hout, int* Wout, Act* final_override,
                       int final_c_off) {
    const bool tc = is_tc(ctx->precision);
    const int lo = passes_of(ctx->precision);
    const Half16 half = half_of(ctx->precision);
    char* slots[2] = {slot0, slot1};
    int cur = 0;
    const LayerSpec* fused_first = nullptr;
    Act in;   // empty -> external fp32 input
    int h = H, w = W, rc;
    for (int i = 0; i < n; ++i) {
        const LayerSpec& l = layers[i];
        const bool last_layer = (i == n - 1) && final_override;
        Act out = last_layer ? *final_override : slot_view(slots[cur], slot_elems, l.cout, tc, lo);
        const bool use_tc = tc && l.cin % 64 == 0 && l.cout % 64 == 0 && l.stride == 1;
        const int c_off = last_layer ? final_c_off : 0;
        const bool pool_after = !strcmp(l.name, "conv1_2") || !strcmp(l.name, "conv2_2") || !strcmp(l.name, "conv3_4");
        const bool fuse_pool = use_tc && pool_after && (h % 2 == 0) && (w % 2 == 0) && !tc_tuning().no_pool_fusion;
        // conv1_1 + conv1_2 as one launch where tc_conv_can_fuse_first() allows it (never in the sm_90a build): layer 0 is skipped
        // here and handed to layer 1
        if (tc && i == 0 && n > 1 && l.cin == 3 && l.cout == 64 && l.k == 3 && l.stride == 1 &&
            !strcmp(layers[1].name, "conv1_2") && (h % 2 == 0) && (w % 2 == 0) && !tc_tuning().no_pool_fusion &&
            tc_conv_can_fuse_first(h, w, layers[1].cin, layers[1].cout, layers[1].k, lo, 1)) {
            fused_first = &layers[0];
            continue;
        }
        if (use_tc && fused_first) {
            rc = add_tc(ctx, pl, scope, l, B, h, w, Split(), 64, l.cin, {}, out.s, out.C, c_off, nullptr, 0, 0, fuse_pool ? 1 : 0, 0, true, fused_first);
            fused_first = nullptr;
        } else if (use_tc) {
            rc = add_tc(ctx, pl, scope, l, B, h, w, in.s, in.C, l.cin, {}, out.s, out.C, c_off, nullptr, 0, 0, fuse_pool ? 1 : 0, 0, true);
        } else if (tc) {   // first layer (Cin = 3): CUDA-core conv writing the split planes directly
            rc = add_direct(ctx, pl, scope, l, B, h, w, in.f, i == 0 ? l.cin : in.C, 0, nullptr, 0, 0, out.s, out.C, c_off);
        } else {
            rc = add_direct(ctx, pl, scope, l, B, h, w, in.f, i == 0 ? l.cin : in.C, 0, out.f, out.C, c_off, Split(), 0, 0);
        }
        if (rc) return rc;
        in = out; cur ^= 1;
        if (fuse_pool) { h /= 2; w /= 2; }
        else if (pool_after) {
            Act pooled = slot_view(slots[cur], slot_elems, l.cout, tc, lo);
            const Act src = in;
            const int hh = h, ww = w, cc = l.cout;
            if (tc && lo == 4) { set_error("fp16_f8c: max-pool must be fused into the convolution (even H, W required)"); return H3D_EINVAL; }
            if (tc) pl->steps.push_back([=](const Ext&, cudaStream_t s) { return launch_maxpool_split(src.s, pooled.s, B, hh, ww, cc, half, s); });
            else pl->steps.push_back([=](const Ext&, cudaStream_t s) { return launch_maxpool_f32(src.f, pooled.f, B, hh, ww, cc, s); });
            pl->launches.push_back(1);
            in = pooled; cur ^= 1; h /= 2; w /= 2;
        }
    }
    *last = in; *Hout = h; *Wout = w;
    return H3D_OK;
}

static int build_handsegnet(h3d_ctx* ctx, int B, int H, int W) {
    H3D_REQUIRE(H % 8 == 0 && W % 8 == 0, "HandSegNet: H and W must be multiples of 8 (got %dx%d)", H, W);
    auto pl = std::make_unique<StagePlan>();
    pl->B = B; pl->H = H; pl->W = W;
    const bool tc = is_tc(ctx->precision);
    if (tc) { if (int rc0 = begin_chain_sync(pl.get(), B)) return rc0; }
    char* r = ctx->ws + ctx->lay.seg_off;
    const int64_t se = slot_elems_seg(B, H, W);
    char* slot0 = r; char* slot1 = r + align_up(se * 4, 1024);
    Act last; int h, w, rc;
    if ((rc = build_trunk(ctx, pl.get(), "HandSegNet", kHandSeg, 14, B, H, W, slot0, slot1, se, &last, &h, &w, nullptr, 0))) return rc;
    // conv6_1 (1x1, 128 -> 512, leaky) and the score-map head conv6_2 (1x1, 512 -> 2, linear; N padded to 64 on the tensor path)
    char* other = (last.f ? (char*)last.f : (char*)last.s.hi) == slot0 ? slot1 : slot0;
    float* low = ctx->lay.seg_low;
    if (tc) {
        Act mid = slot_view(other, (int64_t)B * h * w * 512, 512, true, passes_of(ctx->precision));
        if ((rc = add_tc(ctx, pl.get(), "HandSegNet", kHandSeg[14], B, h, w, last.s, last.C, 128, {}, mid.s, 512, 0, nullptr, 0, 0, 0, 0, true))) return rc;
        if ((rc = add_tc(ctx, pl.get(), "HandSegNet", kHandSeg[15], B, h, w, mid.s, 512, 512, {}, Split(), 0, 0, low, 2, 0, 0, 0, true))) return rc;
    } else {
        float* f512 = (float*)other;
        if ((rc = add_direct(ctx, pl.get(), "HandSegNet", kHandSeg[14], B, h, w, last.f, last.C, 0, f512, 512, 0, Split(), 0, 0))) return rc;
        if ((rc = add_direct(ctx, pl.get(), "HandSegNet", kHandSeg[15], B, h, w, f512, 512, 0, low, 2, 0, Split(), 0, 0))) return rc;
    }
    // e.out == nullptr (pipeline): the x8 up-sampling is fused into the mask post-processing (launch_seg_postprocess reads seg_low)
    pl->steps.push_back([=](const Ext& e, cudaStream_t s) { return e.out ? launch_resize_bilinear_tf1(low, e.out, B, h, w, 2, H, W, s) : H3D_OK; });
    pl->launches.push_back(1);
    ctx->seg = std::move(pl);
    return H3D_OK;
}

static int build_posenet(h3d_ctx* ctx, int B, int Hc, int Wc) {
    H3D_REQUIRE(Hc % 8 == 0 && Wc % 8 == 0, "PoseNet2D: crop height/width must be multiples of 8 (got %dx%d)", Hc, Wc);
    H3D_REQUIRE(Hc <= std::max(ctx->lay.H, 256) && Wc <= std::max(ctx->lay.W, 256), "PoseNet2D: crop %dx%d exceeds the workspace layout", Hc, Wc);
    auto pl = std::make_unique<StagePlan>();
    pl->B = B; pl->H = Hc; pl->W = Wc;
    const bool tc = is_tc(ctx->precision);
    if (tc) { if (int rc0 = begin_chain_sync(pl.get(), B)) return rc0; }
    const int lo = passes_of(ctx->precision);
    const int h8 = Hc / 8, w8 = Wc / 8;
    const int LH = std::max(ctx->lay.H, 256), LW = std::max(ctx->lay.W, 256);
    char* r = ctx->ws + ctx->lay.pose_off;
    const int64_t se = (int64_t)B * Hc * Wc * 64;
    char* slot0 = r; r += align_up((int64_t)B * LH * LW * 64 * 4, 1024);
    char* slot1 = r; r += align_up((int64_t)B * LH * LW * 64 * 4, 1024);
    char* cbuf = r; r += 2 * align_up((int64_t)B * (LH / 8) * (LW / 8) * 192 * 4, 1024);
    float* f512 = (float*)r;
    const int64_t pix = (int64_t)B * h8 * w8;
    int rc, h, w;
    Act last;
    // concat buffer: tensor-core modes = split planes [pix,192] ordered (encoding 0..127 | scoremap 128..148 | zero pad);
    // fp32 mode = [pix,149] in the reference order (scoremap 0..20 | encoding 21..148)   (nets/...:210)
    Act cb;
    if (tc) cb = slot_view(cbuf, pix * 192, 192, true, lo);
    else { cb.C = 149; cb.f = (float*)cbuf; }
    if (tc) {
        const Split cs = cb.s; const size_t bytes = (size_t)pix * 192 * 2;
        pl->steps.push_back([=](const Ext&, cudaStream_t s) {   // zero the padding channels (and everything else) once per call
            H3D_CUDA(cudaMemsetAsync(cs.hi, 0, bytes, s));
            if (cs.lo) H3D_CUDA(cudaMemsetAsync(cs.lo, 0, bytes, s));
            if (cs.l8) { H3D_CUDA(cudaMemsetAsync(cs.l8, 0, bytes / 2, s)); H3D_CUDA(cudaMemsetAsync(cs.h8, 0, bytes / 2, s)); }
            return H3D_OK;
        });
        pl->launches.push_back(0);
    }
    if ((rc = build_trunk(ctx, pl.get(), "PoseNet2D", kPoseTrunk, 15, B, Hc, Wc, slot0, slot1, se, &last, &h, &w, &cb, tc ? 0 : 21))) return rc;
    float** S = ctx->lay.s;
    const Half16 half = half_of(ctx->precision);
    auto head = [&](const char* n6, const char* n7, int cin6, float* sm_out, bool feed_back, const Act& in6) -> int {
        // 1x1 conv (cin6 -> 512 or 128, leaky) then 1x1 conv (-> 21, linear); score-map also fed back into the concat buffer
        LayerSpec l6{n6, 1, 1, 128, cin6, 1}, l7{n7, 1, 1, cin6, 21, 0};
        int rc2;
        if (tc) {
            Act mid = slot_view((char*)f512, pix * cin6, cin6, true, lo);
            if ((rc2 = add_tc(ctx, pl.get(), "PoseNet2D", l6, B, h, w, in6.s, in6.C, 128, {}, mid.s, cin6, 0, nullptr, 0, 0, 0, 0, true))) return rc2;
            rc2 = add_tc(ctx, pl.get(), "PoseNet2D", l7, B, h, w, mid.s, cin6, cin6, {}, feed_back ? cb.s : Split(), 192, 128, sm_out, 21, 0, 0, 0, true);
        } else {
            if ((rc2 = add_direct(ctx, pl.get(), "PoseNet2D", l6, B, h, w, in6.f, in6.C, in6.f == cb.f ? 21 : 0, f512, cin6, 0, Split(), 0, 0))) return rc2;
            rc2 = add_direct(ctx, pl.get(), "PoseNet2D", l7, B, h, w, f512, cin6, 0, sm_out, 21, 0, Split(), 0, 0);
        }
        if (rc2) return rc2;
        if (!tc && feed_back) {
            float* dst = cb.f;
            pl->steps.push_back([=](const Ext&, cudaStream_t s) { return launch_copy_channels(sm_out, dst, pix, 21, 149, 0, s); });
            pl->launches.push_back(1);
        }
        return H3D_OK;
    };
    if ((rc = head("conv5_1", "conv5_2", 512, S[0], true, cb))) return rc;
    std::vector<int> perm(192, -1);
    for (int j = 0; j < 128; ++j) perm[j] = 21 + j;
    for (int j = 0; j < 21; ++j) perm[128 + j] = j;
    char* slots[2] = {slot0, slot1};
    for (int u = 6; u <= 7; ++u) {
        char nm[7][16];
        for (int i = 0; i < 7; ++i) snprintf(nm[i], 16, "conv%d_%d", u, i + 1);
        Act in = cb;
        for (int i = 0; i < 5; ++i) {
            LayerSpec l{nm[i], 7, 1, i == 0 ? 149 : 128, 128, 1};
            Act out = slot_view(slots[i & 1], pix * 128, 128, tc, lo);
            if (tc) rc = add_tc(ctx, pl.get(), "PoseNet2D", l, B, h, w, in.s, in.C, i == 0 ? 192 : 128, i == 0 ? perm : std::vector<int>(), out.s, 128, 0, nullptr, 0, 0, 0, 0, true);
            else rc = add_direct(ctx, pl.get(), "PoseNet2D", l, B, h, w, in.f, in.C, 0, out.f, 128, 0, Split(), 0, 0);
            if (rc) return rc;
            in = out;
        }
        if ((rc = head(nm[5], nm[6], 128, S[u - 5], u == 6, in))) return rc;
    }
    (void)half;
    ctx->pose = std::move(pl);
    return H3D_OK;
}

static int ensure_vp_heads(h3d_ctx* ctx) {
    if (ctx->vp_head_w) return H3D_OK;
    const char* nm[3] = {"ViewpointNet/fc_vp_ux", "ViewpointNet/fc_vp_uy", "ViewpointNet/fc_vp_uz"};
    std::vector<float> w(128 * 3), b(3);
    for (int j = 0; j < 3; ++j) {
        auto wi = ctx->host_w.find(std::string(nm[j]) + "/weights"), bi = ctx->host_w.find(std::string(nm[j]) + "/biases");
        if (wi == ctx->host_w.end() || bi == ctx->host_w.end()) { set_error("weights %s not loaded", nm[j]); return H3D_EWEIGHTS; }
        for (int i = 0; i < 128; ++i) w[i * 3 + j] = wi->second.data[i];
        b[j] = bi->second.data[0];
    }
    HostTensor hw; hw.data = w; hw.shape = {128, 3};
    HostTensor hb; hb.data = b; hb.shape = {3};
    ctx->host_w["ViewpointNet/fc_vp_heads/weights"] = hw;      // fused ux | uy | uz heads: one 128 -> 3 layer of the FC chain
    ctx->host_w["ViewpointNet/fc_vp_heads/biases"] = hb;
    H3D_CUDA(cudaMalloc(&ctx->vp_head_w, w.size() * 4)); H3D_CUDA(cudaMalloc(&ctx->vp_head_b, b.size() * 4));
    H3D_CUDA(cudaMemcpy(ctx->vp_head_w, w.data(), w.size() * 4, cudaMemcpyHostToDevice));
    H3D_CUDA(cudaMemcpy(ctx->vp_head_b, b.data(), b.size() * 4, cudaMemcpyHostToDevice));
    return H3D_OK;
}

static int add_fc(h3d_ctx* ctx, StagePlan* pl, const std::string& name, const float* x, float* y, float* scratch, int64_t scratch_floats,
                  int B, int in_f, int out_f, int leaky) {
    const float *w, *b;
    int rc;
    if ((rc = dev_weight(ctx, name + "/weights", &w))) return rc;
    if ((rc = dev_weight(ctx, name + "/biases", &b))) return rc;
    pl->steps.push_back([=](const Ext&, cudaStream_t s) { return launch_fc(x, w, b, y, scratch, scratch_floats, B, in_f, out_f, leaky, in_f, s); });
    pl->launches.push_back(2);
    pl->flops += 2ll * B * in_f * out_f;
    tag(pl, KIND_FC, 2ll * B * in_f * out_f);
    return H3D_OK;
}

// PosePrior (+ ViewpointNet for the 'proposed' variant): two 6-layer stride-1 / stride-2 conv pyramids on the 32x32 score map
// and their FC stacks.  With a 3-pass tensor-core precision the pyramids run on the wgmma kernel (stride 2 = odd pixels of
// the stride-1 result, Cin / Cout padded to 64 with zero channels); otherwise on the fp32 CUDA-core kernel.  The two networks
// are independent until the final rotation, so ViewpointNet is put on the context's side stream.
static int build_lifting(h3d_ctx* ctx, int B, int variant) {
    auto pl = std::make_unique<StagePlan>();
    pl->B = B; pl->variant = variant;
    Arena a; a.base = ctx->ws + ctx->lay.lift_off;
    // the lifting stage is 0.15 % of the FLOPs: on the tensor path it always runs 3-pass (hi / lo planes), also in the single-pass
    // modes, whose error budget (1e-2) is spent on the trunks; the fp8-correction mode keeps the fp32 CUDA-core kernels
    const int passes = 3;
    const Half16 half = half_of(ctx->precision);
    const bool tc_lift = is_tc(ctx->precision) && passes_of(ctx->precision) != 4 && !tc_tuning().lift_direct;
    const int64_t slot_bytes = align_up((int64_t)B * 32 * 32 * 64 * 4, 1024);
    char* slot_in = a.alloc<char>(slot_bytes);
    const int64_t fcs_floats = lift_fc_scratch_floats(B);
    struct Branch { char* slot[2]; float *xcat, *t1, *t2, *t3, *fcs, *cvs; } br[2];
    for (auto& b : br) {
        b.slot[0] = a.alloc<char>(slot_bytes); b.slot[1] = a.alloc<char>(slot_bytes);
        b.xcat = a.alloc<float>((int64_t)B * 4100);
        b.t1 = a.alloc<float>((int64_t)B * 512); b.t2 = a.alloc<float>((int64_t)B * 512); b.t3 = a.alloc<float>((int64_t)B * 64);
        b.fcs = a.alloc<float>(fcs_floats);
        b.cvs = a.alloc<float>(kConvSplitKScratchFloats);
    }
    float* can = a.alloc<float>((int64_t)B * 63);
    float* uxyz = a.alloc<float>((int64_t)B * 4);
    H3D_REQUIRE(ctx->lay.lift_off + a.off <= ctx->lay.total, "lifting workspace region too small (internal error)");
    int rc;
    Act xin;   // tensor-core path: the 21-channel score map as split planes with 64 channels (43 zero)
    if (tc_lift) {
        xin = slot_view(slot_in, (int64_t)B * 32 * 32 * 64, 64, true, passes);
        const Split xs = xin.s;
        pl->steps.push_back([=](const Ext& e, cudaStream_t s) { return launch_f32_to_split(e.in, xs, (int64_t)B * 32 * 32, 21, 64, half, s); });
        pl->launches.push_back(1);
        pl->seal();
    }
    // returns the flattened NHWC fp32 feature map [B, 4*4*C] in *feat
    auto pyramid = [&](const std::string& scope, const LayerSpec* L, const Branch& b, float** feat) -> int {
        int h = 32, w = 32;
        if (!tc_lift) {
            float* bufs[2] = {(float*)b.slot[0], (float*)b.slot[1]};
            const float* in = nullptr; int cin_total = 21;
            for (int i = 0; i < 6; ++i) {
                float* out = bufs[i & 1];
                int rc2 = add_direct(ctx, pl.get(), scope, L[i], B, h, w, in, cin_total, 0, out, L[i].cout, 0, Split(), 0, 0, b.cvs);
                if (rc2) return rc2;
                h = ceil_div(h, L[i].stride); w = ceil_div(w, L[i].stride);
                in = out; cin_total = L[i].cout;
            }
            *feat = bufs[1];
            return H3D_OK;
        }
        Act in = xin;
        for (int i = 0; i < 6; ++i) {
            const LayerSpec& l = L[i];
            const int Cin_pad = (int)align_up(l.cin, 64), Cout_pad = (int)align_up(l.cout, 64);
            const int ho = h / l.stride, wo = w / l.stride;
            const bool last = i == 5;
            Act out = slot_view(b.slot[i & 1], (int64_t)B * ho * wo * Cout_pad, Cout_pad, true, passes);
            float* yf = last ? (float*)b.slot[i & 1] : nullptr;
            int rc2 = add_tc(ctx, pl.get(), scope, l, B, h, w, in.s, in.C, Cin_pad, {}, last ? Split() : out.s, Cout_pad, 0, yf, l.cout, 0,
                             l.stride == 2 ? 2 : 0, passes);
            if (rc2) return rc2;
            if (last) *feat = yf;
            h = ho; w = wo; in = out;
        }
        return H3D_OK;
    };
    // ---- PosePrior on the caller's stream (nets/ColorHandPose3DNetwork.py:249-272; bottleneck nets/PosePriorNetwork.py:113-116)
    const bool bott = variant == H3D_VARIANT_BOTTLENECK;
    auto xyz = ctx->host_w.find("PosePrior/fc_xyz/weights");
    if (xyz == ctx->host_w.end()) { set_error("weights PosePrior/fc_xyz not loaded"); return H3D_EWEIGHTS; }
    const int xyz_in = (int)xyz->second.shape[0];
    // FC layers on the tensor-core kernel: a fully connected layer is a 1x1 convolution over B "images" of 1x1 pixels (tile =
    // 128 batch rows, K = in_features padded to 64, weights [in,out] = HWIO [1,1,in,out]); activations stay split planes
    struct Planes { Split s; int stride; };
    auto carve_planes = [&](char*& cur, int width) -> Planes {
        Planes pz; pz.stride = (int)align_up(width, 64);
        const int64_t bytes = align_up((int64_t)B * pz.stride * 2, 1024);
        pz.s.hi = (uint16_t*)cur; pz.s.lo = (uint16_t*)(cur + bytes);
        cur += 2 * bytes;
        return pz;
    };
    auto fc_tc = [&](const std::string& scope, const char* name, int in_f, int out_f, int leaky, const Planes& x, const Planes* y, float* yf) -> int {
        LayerSpec l{name, 1, 1, in_f, out_f, leaky};
        return add_tc(ctx, pl.get(), scope, l, B, 1, 1, x.s, x.stride, (int)align_up(in_f, 64), {}, y ? y->s : Split(), y ? y->stride : 0, 0, yf,
                      out_f, 0, 0, passes);
    };
    // ---- FC stacks + Rodrigues / flip / rotate as ONE kernel (fc_chain_kernel): both pyramids first (ViewpointNet on the side
    //      stream), their concat kernels, one join, one launch.  tune.fc_chain = 0 keeps the layer-by-layer path below.
    const bool use_chain = tc_lift && tc_tuning().fc_chain != 0;
    if (use_chain) {
        if (bott) H3D_REQUIRE(xyz_in == 30, "bottleneck variant needs PosePrior/fc_xyz/weights of shape [30,63]");
        else H3D_REQUIRE(xyz_in == 512, "PosePrior/fc_xyz/weights must have shape [512,63] for this variant");
        FcChainDesc chains[2];
        int64_t fl = 0;
        auto fc_layer = [&](FcChainDesc& cd, const std::string& scope, const char* name, int in_f, int out_f, int leaky, const Planes& x, const Planes* y,
                            float* yf, int yf_stride) -> int {
            LayerSpec l{name, 1, 1, in_f, out_f, leaky};
            const PackedW* pw;
            int rc2 = get_packed(ctx, scope, l, (int)align_up(in_f, 64), {}, &pw, passes);
            if (rc2) return rc2;
            FcLayerDesc& d = cd.layer[cd.num_layers++];
            d.x = x.s; d.x_stride = x.stride; d.in_features = in_f;
            d.w = pw->w; d.bias = pw->bias; d.w_scale = pw->w_scale; d.out_features = out_f; d.out_pad = pw->Cout_pad;
            d.y = y ? y->s : Split(); d.y_stride = y ? y->stride : 0; d.yf = yf; d.yf_stride = yf_stride; d.leaky = leaky;
            fl += 2ll * B * in_f * out_f;
            return H3D_OK;
        };
        const bool proposed = variant == H3D_VARIANT_PROPOSED;
        if (proposed) {
            if ((rc = ensure_vp_heads(ctx))) return rc;
            const Branch& b = br[1];
            float* feat = nullptr;
            pl->cur_lane = 1;
            if ((rc = pyramid("ViewpointNet", kViewpoint, b, &feat))) return rc;
            char* cur = b.slot[0];
            const Planes xp = carve_planes(cur, 4098), p1 = carve_planes(cur, 256), p2 = carve_planes(cur, 128);
            pl->steps.push_back([=](const Ext& e, cudaStream_t s) { return launch_concat_handside_split(feat, e.hand_side, xp.s, B, 4096, xp.stride, half, s); });
            pl->launches.push_back(1);
            pl->seal();
            pl->cur_lane = 0;
            if ((rc = fc_layer(chains[1], "ViewpointNet", "fc_vp0", 4098, 256, 1, xp, &p1, nullptr, 0))) return rc;
            if ((rc = fc_layer(chains[1], "ViewpointNet", "fc_vp1", 256, 128, 1, p1, &p2, nullptr, 0))) return rc;
            if ((rc = fc_layer(chains[1], "ViewpointNet", "fc_vp_heads", 128, 3, 0, p2, nullptr, uxyz, 3))) return rc;    // ux | uy | uz (:303-308)
        }
        {
            const Branch& b = br[0];
            float* feat = nullptr;
            if ((rc = pyramid("PosePrior", kPosePrior, b, &feat))) return rc;
            char* cur = b.slot[0];
            const Planes xp = carve_planes(cur, 2050), p1 = carve_planes(cur, 512), p2 = carve_planes(cur, 512), p3 = carve_planes(cur, 64);
            pl->steps.push_back([=](const Ext& e, cudaStream_t s) { return launch_concat_handside_split(feat, e.hand_side, xp.s, B, 2048, xp.stride, half, s); });
            pl->launches.push_back(1);
            if ((rc = fc_layer(chains[0], "PosePrior", "fc_rel0", 2050, 512, 1, xp, &p1, nullptr, 0))) return rc;
            if ((rc = fc_layer(chains[0], "PosePrior", "fc_rel1", 512, 512, 1, p1, &p2, nullptr, 0))) return rc;
            if (bott) {
                if ((rc = fc_layer(chains[0], "PosePrior", "fc_bottleneck", 512, 30, 0, p2, &p3, nullptr, 0))) return rc;
                if ((rc = fc_layer(chains[0], "PosePrior", "fc_xyz", 30, 63, 0, p3, nullptr, can, 63))) return rc;
            } else {
                if ((rc = fc_layer(chains[0], "PosePrior", "fc_xyz", 512, 63, 0, p2, nullptr, can, 63))) return rc;
            }
            pl->seal();
        }
        FcChainPlan* fp = fc_chain_plan_create(chains, proposed ? 2 : 1, B, half, can, uxyz, ctx->fc_counter, ctx->err_flag);
        if (!fp) return H3D_ECUDA;
        pl->fc.push_back(fp);
        const int var = variant;
        pl->steps.push_back([=](const Ext& e, cudaStream_t s) {
            int rc2 = fc_chain_launch(fp, e.hand_side, var == H3D_VARIANT_PROPOSED ? e.out3 : nullptr, var == H3D_VARIANT_PROPOSED ? e.out : nullptr, s);
            if (rc2) return rc2;
            if (var == H3D_VARIANT_LOCAL) {
                if (e.out2) H3D_CUDA(cudaMemcpyAsync(e.out2, can, (size_t)B * 63 * 4, cudaMemcpyDeviceToDevice, s));
                return launch_bone_rel_trafo_inv(can, e.out, B, s);     // nets/PosePriorNetwork.py:70-75
            }
            if (var != H3D_VARIANT_PROPOSED) H3D_CUDA(cudaMemcpyAsync(e.out, can, (size_t)B * 63 * 4, cudaMemcpyDeviceToDevice, s));
            if (e.out2) H3D_CUDA(cudaMemcpyAsync(e.out2, can, (size_t)B * 63 * 4, cudaMemcpyDeviceToDevice, s));
            return H3D_OK;
        });
        pl->launches.push_back(variant == H3D_VARIANT_LOCAL ? 2 : 1);
        pl->flops += fl;
        tag(pl.get(), KIND_TC, fl);
        pl->seal(true);                                       // joins the ViewpointNet branch before the launch
        ctx->lift = std::move(pl);
        return H3D_OK;
    }
    auto pose_prior = [&]() -> int {
        const Branch& b = br[0];
        float* feat = nullptr;
        int rc2;
        if ((rc2 = pyramid("PosePrior", kPosePrior, b, &feat))) return rc2;
        if (bott) H3D_REQUIRE(xyz_in == 30, "bottleneck variant needs PosePrior/fc_xyz/weights of shape [30,63]");
        else H3D_REQUIRE(xyz_in == 512, "PosePrior/fc_xyz/weights must have shape [512,63] for this variant");
        if (tc_lift) {   // slot[0] (layer-4 output, dead by now) holds the FC activations
            char* cur = b.slot[0];
            const Planes xp = carve_planes(cur, 2050), p1 = carve_planes(cur, 512), p2 = carve_planes(cur, 512), p3 = carve_planes(cur, 64);
            pl->steps.push_back([=](const Ext& e, cudaStream_t s) { return launch_concat_handside_split(feat, e.hand_side, xp.s, B, 2048, xp.stride, half, s); });
            pl->launches.push_back(1);
            if ((rc2 = fc_tc("PosePrior", "fc_rel0", 2050, 512, 1, xp, &p1, nullptr))) return rc2;
            if ((rc2 = fc_tc("PosePrior", "fc_rel1", 512, 512, 1, p1, &p2, nullptr))) return rc2;
            if (bott) {
                if ((rc2 = fc_tc("PosePrior", "fc_bottleneck", 512, 30, 0, p2, &p3, nullptr))) return rc2;
                return fc_tc("PosePrior", "fc_xyz", 30, 63, 0, p3, nullptr, can);
            }
            return fc_tc("PosePrior", "fc_xyz", 512, 63, 0, p2, nullptr, can);
        }
        float* xcat = b.xcat;
        pl->steps.push_back([=](const Ext& e, cudaStream_t s) { return launch_concat_handside(feat, e.hand_side, xcat, B, 2048, s); });
        pl->launches.push_back(1);
        if ((rc2 = add_fc(ctx, pl.get(), "PosePrior/fc_rel0", b.xcat, b.t1, b.fcs, fcs_floats, B, 2050, 512, 1))) return rc2;
        if ((rc2 = add_fc(ctx, pl.get(), "PosePrior/fc_rel1", b.t1, b.t2, b.fcs, fcs_floats, B, 512, 512, 1))) return rc2;
        if (bott) {
            if ((rc2 = add_fc(ctx, pl.get(), "PosePrior/fc_bottleneck", b.t2, b.t3, b.fcs, fcs_floats, B, 512, 30, 0))) return rc2;
            if ((rc2 = add_fc(ctx, pl.get(), "PosePrior/fc_xyz", b.t3, can, b.fcs, fcs_floats, B, 30, 63, 0))) return rc2;
        } else {
            if ((rc2 = add_fc(ctx, pl.get(), "PosePrior/fc_xyz", b.t2, can, b.fcs, fcs_floats, B, 512, 63, 0))) return rc2;
        }
        return H3D_OK;
    };
    if (variant == H3D_VARIANT_PROPOSED) {
        // ---- ViewpointNet on the side stream (nets/ColorHandPose3DNetwork.py:274-309), enqueued first so that both branches
        //      are in flight while the host builds the second one
        if ((rc = ensure_vp_heads(ctx))) return rc;
        const Branch& b = br[1];
        float* feat = nullptr;
        pl->cur_lane = 1;
        if ((rc = pyramid("ViewpointNet", kViewpoint, b, &feat))) return rc;
        if (tc_lift) {
            char* cur = b.slot[0];
            const Planes xp = carve_planes(cur, 4098), p1 = carve_planes(cur, 256);
            pl->steps.push_back([=](const Ext& e, cudaStream_t s) { return launch_concat_handside_split(feat, e.hand_side, xp.s, B, 4096, xp.stride, half, s); });
            pl->launches.push_back(1);
            if ((rc = fc_tc("ViewpointNet", "fc_vp0", 4098, 256, 1, xp, &p1, nullptr))) return rc;
            if ((rc = fc_tc("ViewpointNet", "fc_vp1", 256, 128, 1, p1, nullptr, b.t2))) return rc;   // fp32 [B,128] for the three 128 -> 1 heads
        } else {
            float* xcat = b.xcat;
            pl->steps.push_back([=](const Ext& e, cudaStream_t s) { return launch_concat_handside(feat, e.hand_side, xcat, B, 4096, s); });
            pl->launches.push_back(1);
            if ((rc = add_fc(ctx, pl.get(), "ViewpointNet/fc_vp0", b.xcat, b.t1, b.fcs, fcs_floats, B, 4098, 256, 1))) return rc;
            if ((rc = add_fc(ctx, pl.get(), "ViewpointNet/fc_vp1", b.t1, b.t2, b.fcs, fcs_floats, B, 256, 128, 1))) return rc;
        }
        const float* hw = ctx->vp_head_w; const float* hb = ctx->vp_head_b;
        float* t2 = b.t2; float* fcs = b.fcs;
        pl->steps.push_back([=](const Ext&, cudaStream_t s) { return launch_fc(t2, hw, hb, uxyz, fcs, fcs_floats, B, 128, 3, 0, 128, s); });
        pl->launches.push_back(2);
        tag(pl.get(), KIND_FC, 2ll * B * 128 * 3);
        pl->seal();
        pl->cur_lane = 0;
    }
    if ((rc = pose_prior())) return rc;
    pl->seal();
    if (variant == H3D_VARIANT_PROPOSED) {
        // Rodrigues / flip / rotate (:239-247,311-334): needs both branches
        pl->steps.push_back([=](const Ext& e, cudaStream_t s) {
            if (e.out2) H3D_CUDA(cudaMemcpyAsync(e.out2, can, (size_t)B * 63 * 4, cudaMemcpyDeviceToDevice, s));
            return launch_rotate_canonical(can, uxyz, e.hand_side, B, e.out3, e.out, s);
        });
        pl->launches.push_back(1);
        pl->seal(true);
    } else if (variant == H3D_VARIANT_LOCAL) {
        // nets/PosePriorNetwork.py:70-75: the network predicts bone-relative coordinates; assemble xyz by forward kinematics
        pl->steps.push_back([=](const Ext& e, cudaStream_t s) {
            if (e.out2) H3D_CUDA(cudaMemcpyAsync(e.out2, can, (size_t)B * 63 * 4, cudaMemcpyDeviceToDevice, s));
            return launch_bone_rel_trafo_inv(can, e.out, B, s);
        });
        pl->launches.push_back(1);
        pl->seal();
    } else {
        pl->steps.push_back([=](const Ext& e, cudaStream_t s) {
            H3D_CUDA(cudaMemcpyAsync(e.out, can, (size_t)B * 63 * 4, cudaMemcpyDeviceToDevice, s));
            if (e.out2) H3D_CUDA(cudaMemcpyAsync(e.out2, can, (size_t)B * 63 * 4, cudaMemcpyDeviceToDevice, s));
            return H3D_OK;
        });
        pl->launches.push_back(0);
        pl->seal();
    }
    ctx->lift = std::move(pl);
    return H3D_OK;
}

static int run_plan(h3d_ctx* ctx, StagePlan* pl, const Ext& e, cudaStream_t s) {
    bool forked = false;
    auto join = [&]() -> int {
        if (!forked) return H3D_OK;
        H3D_CUDA(cudaEventRecord(ctx->ev_join, ctx->side));
        H3D_CUDA(cudaStreamWaitEvent(s, ctx->ev_join, 0));
        forked = false;
        return H3D_OK;
    };
    const bool lanes = !tc_tuning().no_side_stream;
    for (size_t i = 0; i < pl->steps.size(); ++i) {
        int rc;
        const int ln = (lanes && i < pl->lane.size()) ? pl->lane[i] : 0;
        if (i < pl->join_before.size() && pl->join_before[i] && (rc = join())) return rc;
        if (ln == 1 && !forked) {   // the branch starts from everything enqueued on the caller's stream so far
            H3D_CUDA(cudaEventRecord(ctx->ev_fork, s));
            H3D_CUDA(cudaStreamWaitEvent(ctx->side, ctx->ev_fork, 0));
            forked = true;
        }
        cudaStream_t st = ln == 1 ? ctx->side : s;
        h3d_ctx::ProfRec pr;
        const bool prof = ctx->profiling && pl->launches[i] > 0;
        if (prof) {
            H3D_CUDA(cudaEventCreate(&pr.a)); H3D_CUDA(cudaEventCreate(&pr.b));
            pr.kind = i < pl->kinds.size() ? pl->kinds[i] : KIND_OTHER;
            pr.flops = i < pl->step_flops.size() ? pl->step_flops[i] : 0;
            H3D_CUDA(cudaEventRecord(pr.a, st));
        }
        rc = pl->steps[i](e, st);
        if (rc) { join(); return rc; }
        if (prof) { H3D_CUDA(cudaEventRecord(pr.b, st)); ctx->prof.push_back(pr); }
        ctx->launches += pl->launches[i];
    }
    return join();
}

static int check_device() {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        cudaGetLastError();
        set_error("no CUDA device available (%s): hand3d_b200 has no CPU fallback", e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
        return H3D_ENODEVICE;
    }
    return H3D_OK;
}

}  // namespace h3d

// =============================================================================================== C ABI
extern "C" {

const char* h3d_last_error(void) { return g_err; }
int h3d_version(void) { return 100; }

int h3d_device_available(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) { cudaGetLastError(); return 0; }
    cudaDeviceProp p;
    if (cudaGetDeviceProperties(&p, 0) != cudaSuccess) { cudaGetLastError(); return 0; }
    return p.major == 9 && p.minor == 0 ? 1 : 0;
}

int h3d_create(h3d_ctx** out, int device) {
    H3D_REQUIRE(out != nullptr, "h3d_create: out is NULL");
    int rc = check_device();
    if (rc) return rc;
    cudaDeviceProp p;
    H3D_CUDA(cudaGetDeviceProperties(&p, device));
    if (p.major != 9 || p.minor != 0) {
        set_error("device %d (%s) has compute capability %d.%d; hand3d_b200 is built for sm_90a only", device, p.name, p.major, p.minor);
        return H3D_ENODEVICE;
    }
    H3D_CUDA(cudaSetDevice(device));
    h3d_ctx* c = new h3d_ctx();
    c->device = device;
    memset(&c->lay, 0, sizeof(c->lay));
    if (cudaStreamCreateWithFlags(&c->side, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&c->side2, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->ev_fork2, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->ev_join2, cudaEventDisableTiming) != cudaSuccess) {
        set_error("h3d_create: cannot create the side streams (%s)", cudaGetErrorString(cudaGetLastError()));
        h3d_destroy(c);
        return H3D_ECUDA;
    }
    if (cudaHostAlloc((void**)&c->err_flag, sizeof(int), cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) {
        set_error("h3d_create: cannot allocate the error word (%s)", cudaGetErrorString(cudaGetLastError()));
        h3d_destroy(c);
        return H3D_ECUDA;
    }
    *c->err_flag = 0;
    if (cudaMalloc(&c->fc_counter, sizeof(unsigned int)) != cudaSuccess || cudaMemset(c->fc_counter, 0, sizeof(unsigned int)) != cudaSuccess) {
        set_error("h3d_create: cannot allocate the FC-chain ticket (%s)", cudaGetErrorString(cudaGetLastError()));
        h3d_destroy(c);
        return H3D_ECUDA;
    }
    tc_tuning();   // read the H3D_* environment switches now, never on a launch path
    *out = c;
    return H3D_OK;
}

int h3d_check_errors(h3d_ctx* ctx, int* code) {
    H3D_REQUIRE(ctx != nullptr, "h3d_check_errors: ctx is NULL");
    const int c = ctx->err_flag ? *(volatile int*)ctx->err_flag : 0;
    if (code) *code = c;
    if (c == 0) return H3D_OK;
    static const char* what[] = {"", "TMA producer waiting for a free shared-memory stage", "unused wait code",
                                 "wgmma warpgroup waiting for a TMA stage", "unused wait code", "unused wait code"};
    if (c >= 100) set_error("device-side timeout: gather_records_p2p never saw the records of peer rank %d (code %d)", c - 100, c);
    else set_error("device-side timeout in a tensor-core convolution kernel: %s (code %d); the kernel trapped", c >= 1 && c <= 5 ? what[c] : "unknown wait", c);
    return H3D_ECUDA;
}

int h3d_destroy(h3d_ctx* ctx) {
    if (!ctx) return H3D_OK;
    DeviceGuard guard(ctx->device);
    ctx->drop_plans();
    for (auto& kv : ctx->dev_w) cudaFree(kv.second);
    for (auto& kv : ctx->packed) free_packed(kv.second);
    if (ctx->vp_head_w) cudaFree(ctx->vp_head_w);
    if (ctx->vp_head_b) cudaFree(ctx->vp_head_b);
    if (ctx->side) { cudaStreamSynchronize(ctx->side); cudaStreamDestroy(ctx->side); }      // branches always join the caller's stream;
    if (ctx->side2) { cudaStreamSynchronize(ctx->side2); cudaStreamDestroy(ctx->side2); }   // the syncs only matter after a failed call
    for (cudaEvent_t e : {ctx->ev_fork, ctx->ev_join, ctx->ev_fork2, ctx->ev_join2})
        if (e) cudaEventDestroy(e);
    if (ctx->op_scratch) cudaFree(ctx->op_scratch);
    for (void* p : ctx->retired) cudaFree(p);
    if (ctx->err_flag) cudaFreeHost(ctx->err_flag);
    if (ctx->fc_counter) cudaFree(ctx->fc_counter);
    delete ctx;
    return H3D_OK;
}

int h3d_set_precision(h3d_ctx* ctx, int precision) {
    H3D_REQUIRE(ctx && precision >= H3D_PREC_FP32_FFMA && precision <= H3D_PREC_FP16_F8C, "h3d_set_precision: bad argument");
    if (precision != ctx->precision) { ctx->precision = precision; ctx->drop_plans(); }
    return H3D_OK;
}
int h3d_get_precision(const h3d_ctx* ctx) { return ctx ? ctx->precision : H3D_EINVAL; }
int h3d_set_tuning(h3d_ctx* ctx, const char* key, int value) {
    H3D_REQUIRE(key != nullptr, "h3d_set_tuning: key is NULL");
    int rc = tc_set_tuning(key, value);
    if (!rc && ctx) ctx->drop_plans();   // plans bake the kernel choice in
    return rc;
}
int64_t h3d_launch_count(const h3d_ctx* ctx) { return ctx ? ctx->launches : 0; }

int h3d_profile_begin(h3d_ctx* ctx) {
    H3D_REQUIRE(ctx != nullptr, "h3d_profile_begin: ctx is NULL");
    for (auto& r : ctx->prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    ctx->prof.clear();
    ctx->profiling = true;
    return H3D_OK;
}

int h3d_profile_end(h3d_ctx* ctx, double* ms_by_kind, int64_t* flops_by_kind, int64_t* launches_by_kind) {
    H3D_REQUIRE(ctx && ms_by_kind && flops_by_kind && launches_by_kind, "h3d_profile_end: bad argument");
    ctx->profiling = false;
    for (int k = 0; k < KIND_COUNT; ++k) { ms_by_kind[k] = 0; flops_by_kind[k] = 0; launches_by_kind[k] = 0; }
    H3D_CUDA(cudaDeviceSynchronize());
    for (auto& r : ctx->prof) {
        float ms = 0.f;
        H3D_CUDA(cudaEventElapsedTime(&ms, r.a, r.b));
        ms_by_kind[r.kind] += ms; flops_by_kind[r.kind] += r.flops; launches_by_kind[r.kind] += 1;
        cudaEventDestroy(r.a); cudaEventDestroy(r.b);
    }
    ctx->prof.clear();
    return H3D_OK;
}

int h3d_load_weight(h3d_ctx* ctx, const char* name, const float* host_data, const int64_t* shape, int ndim) {
    H3D_REQUIRE(ctx && name && host_data && shape && ndim >= 1 && ndim <= 4, "h3d_load_weight: bad argument");
    auto it = known_vars().find(name);
    if (it == known_vars().end()) { set_error("Unknown variable name: %s", name); return H3D_EWEIGHTS; }
    VarShape vs = it->second;
    const std::string nm(name);
    bool ok = vs.nd == ndim;
    for (int i = 0; ok && i < ndim; ++i) ok = vs.s[i] == shape[i];
    if (!ok && nm == "PosePrior/fc_xyz/weights" && ndim == 2 && shape[0] == 30 && shape[1] == 63) ok = true;   // bottleneck variant
    if (!ok) { set_error("Shape mismatch for variable %s", name); return H3D_EWEIGHTS; }
    int64_t n = 1;
    for (int i = 0; i < ndim; ++i) n *= shape[i];
    if (nm.find("/fc_") != std::string::npos) {   // tf.check_numerics (utils/general.py:122,127)
        for (int64_t i = 0; i < n; ++i)
            if (!std::isfinite(host_data[i])) { set_error("check_numerics: %s contains NaN/Inf", name); return H3D_EWEIGHTS; }
    }
    HostTensor t;
    t.data.assign(host_data, host_data + n);
    t.shape.assign(shape, shape + ndim);
    float* d = nullptr;
    H3D_CUDA(cudaSetDevice(ctx->device));
    H3D_CUDA(cudaMalloc(&d, (size_t)n * 4));
    H3D_CUDA(cudaMemcpy(d, host_data, (size_t)n * 4, cudaMemcpyHostToDevice));
    auto old = ctx->dev_w.find(nm);
    if (old != ctx->dev_w.end()) cudaFree(old->second);
    ctx->dev_w[nm] = d;
    ctx->host_w[nm] = std::move(t);
    // invalidate everything derived from this variable
    const std::string layer = nm.substr(0, nm.rfind('/'));
    for (auto pit = ctx->packed.begin(); pit != ctx->packed.end();) {
        if (pit->first.compare(0, layer.size() + 1, layer + "|") == 0) { free_packed(pit->second); pit = ctx->packed.erase(pit); }
        else ++pit;
    }
    if (nm.find("fc_vp_u") != std::string::npos && ctx->vp_head_w) {
        cudaFree(ctx->vp_head_w); cudaFree(ctx->vp_head_b); ctx->vp_head_w = ctx->vp_head_b = nullptr;
        ctx->host_w.erase("ViewpointNet/fc_vp_heads/weights"); ctx->host_w.erase("ViewpointNet/fc_vp_heads/biases");
        for (auto pit = ctx->packed.begin(); pit != ctx->packed.end();) {
            if (pit->first.compare(0, 25, "ViewpointNet/fc_vp_heads|") == 0) { free_packed(pit->second); pit = ctx->packed.erase(pit); }
            else ++pit;
        }
    }
    ctx->drop_plans();
    return H3D_OK;
}

int h3d_scope_ready(const h3d_ctx* ctx, const char* scope) {
    if (!ctx || !scope) return 0;
    const std::string pre = std::string(scope) + "/";
    int found = 0;
    for (auto& kv : known_vars()) {
        if (kv.first.compare(0, pre.size(), pre) != 0) continue;
        if (kv.first.find("fc_bottleneck") != std::string::npos) continue;
        ++found;
        if (!ctx->host_w.count(kv.first)) return 0;
    }
    return found > 0;
}

int64_t h3d_workspace_bytes(const h3d_ctx* ctx, int B, int H, int W) {
    if (!ctx || B <= 0 || H <= 0 || W <= 0) return H3D_EINVAL;
    h3d_ctx::Layout L;
    layout(L, nullptr, B, H, W);
    return L.total;
}

int h3d_set_workspace(h3d_ctx* ctx, void* dev_ptr, int64_t bytes) {
    H3D_REQUIRE(ctx != nullptr, "h3d_set_workspace: ctx is NULL");
    H3D_REQUIRE(((uintptr_t)dev_ptr & 1023) == 0, "h3d_set_workspace: pointer must be 1024-byte aligned");
    ctx->drop_plans();
    memset(&ctx->lay, 0, sizeof(ctx->lay));
    ctx->ws = (char*)dev_ptr; ctx->ws_bytes = bytes;
    return H3D_OK;
}

// logits == nullptr: stop after the low-resolution head (Layout::seg_low); the caller up-samples (fused into the mask post-processing)
static int run_handsegnet(h3d_ctx* ctx, const float* image, int B, int H, int W, float* logits, void* stream) {
    int rc;
    if ((rc = ensure_layout_covers(ctx, B, H, W, 0, 0))) return rc;
    if (!ctx->seg || ctx->seg->B != B || ctx->seg->H != H || ctx->seg->W != W)
        if ((rc = build_handsegnet(ctx, B, H, W))) return rc;
    Ext e; e.in = image; e.out = logits;
    rc = run_plan(ctx, ctx->seg.get(), e, (cudaStream_t)stream);
    if (!logits) ctx->launches -= 1;   // the skipped up-sampling step
    return rc;
}

int h3d_handsegnet_forward(h3d_ctx* ctx, const float* image, int B, int H, int W, float* logits, void* stream) {
    DeviceGuard guard_(ctx ? ctx->device : 0);
    H3D_REQUIRE(ctx && image && logits && B > 0, "h3d_handsegnet_forward: bad argument");
    return run_handsegnet(ctx, image, B, H, W, logits, stream);
}

int h3d_posenet_forward(h3d_ctx* ctx, const float* image_crop, int B, int Hc, int Wc, float* s0, float* s1, float* s2, void* stream) {
    DeviceGuard guard_(ctx ? ctx->device : 0);
    H3D_REQUIRE(ctx && image_crop && B > 0, "h3d_posenet_forward: bad argument");
    int rc;
    if ((rc = ensure_layout_covers(ctx, B, 0, 0, Hc, Wc))) return rc;
    if (!ctx->pose || ctx->pose->B != B || ctx->pose->H != Hc || ctx->pose->W != Wc)
        if ((rc = build_posenet(ctx, B, Hc, Wc))) return rc;
    Ext e; e.in = image_crop;
    if ((rc = run_plan(ctx, ctx->pose.get(), e, (cudaStream_t)stream))) return rc;
    float* outs[3] = {s0, s1, s2};
    const size_t bytes = (size_t)B * (Hc / 8) * (Wc / 8) * 21 * 4;
    for (int i = 0; i < 3; ++i)
        if (outs[i]) H3D_CUDA(cudaMemcpyAsync(outs[i], ctx->lay.s[i], bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return H3D_OK;
}

int h3d_pose2d_forward(h3d_ctx* ctx, const float* image_crop, int B, int Hc, int Wc, float* keypoints_scoremap, int32_t* keypoints_uv,
                       void* stream) {
    H3D_REQUIRE(ctx && image_crop && B > 0, "h3d_pose2d_forward: bad argument");
    H3D_REQUIRE(keypoints_scoremap || (Hc <= 256 && Wc <= 256), "h3d_pose2d_forward: keypoints_scoremap is required for crops larger than 256x256");
    DeviceGuard guard_(ctx->device);
    cudaStream_t s = (cudaStream_t)stream;
    int rc;
    if ((rc = h3d_posenet_forward(ctx, image_crop, B, Hc, Wc, nullptr, nullptr, nullptr, stream))) return rc;
    h3d_ctx::Layout& L = ctx->lay;
    float* kps = keypoints_scoremap ? keypoints_scoremap : L.kp_scoremap;
    int nl = 0;
    if (keypoints_uv) rc = launch_resize_argmax21(L.s[2], kps, B, Hc / 8, Wc / 8, Hc, Wc, L.argmax_scratch, keypoints_uv, s, &nl);
    else { rc = launch_resize_bilinear_tf1(L.s[2], kps, B, Hc / 8, Wc / 8, 21, Hc, Wc, s); nl = 1; }
    ctx->launches += nl;
    return rc;
}

int h3d_lifting_forward(h3d_ctx* ctx, const float* scoremap32, const float* hand_side, int B, int variant,
                        float* coord_xyz_rel_normed, float* coord_can, float* rot_mat, void* stream) {
    DeviceGuard guard_(ctx ? ctx->device : 0);
    H3D_REQUIRE(ctx && scoremap32 && hand_side && coord_xyz_rel_normed && B > 0, "h3d_lifting_forward: bad argument");
    H3D_REQUIRE(variant >= H3D_VARIANT_DIRECT && variant <= H3D_VARIANT_LOCAL, "h3d_lifting_forward: unknown variant");
    int rc;
    if ((rc = ensure_layout_covers(ctx, B, 0, 0, 0, 0))) return rc;
    if (!ctx->lift || ctx->lift->B != B || ctx->lift->variant != variant)
        if ((rc = build_lifting(ctx, B, variant))) return rc;
    Ext e; e.in = scoremap32; e.hand_side = hand_side; e.out = coord_xyz_rel_normed; e.out2 = coord_can; e.out3 = rot_mat;
    return run_plan(ctx, ctx->lift.get(), e, (cudaStream_t)stream);
}

int h3d_pipeline_forward(h3d_ctx* ctx, const float* image, const float* hand_side, int B, int H, int W, int with_pose3d,
                         const float* force_center, const float* force_scale, float* hand_scoremap, float* image_crop,
                         float* scale_crop, float* center, float* keypoints_scoremap, float* keypoint_coord3d,
                         int32_t* keypoints_uv, uint8_t* hand_mask, void* stream) {
    DeviceGuard guard_(ctx ? ctx->device : 0);
    H3D_REQUIRE(ctx && image && B > 0, "h3d_pipeline_forward: bad argument");
    H3D_REQUIRE(!with_pose3d || (hand_side && keypoint_coord3d), "h3d_pipeline_forward: hand_side / keypoint_coord3d required with pose3d");
    cudaStream_t s = (cudaStream_t)stream;
    int rc;
    if ((rc = ensure_layout_covers(ctx, B, H, W, 256, 256))) return rc;
    h3d_ctx::Layout& L = ctx->lay;
    float* seg = hand_scoremap ? hand_scoremap : L.hand_scoremap;
    float* crop = image_crop ? image_crop : L.image_crop;
    float* kps = keypoints_scoremap ? keypoints_scoremap : L.kp_scoremap;
    float* cen = center ? center : L.center;
    float* scl = scale_crop ? scale_crop : L.scale;
    // HandSegNet (nets/...:78-79)
    // (its x8 up-sampling, nets/...:166, is fused into the next kernel: the 0.82 MB / image hand_scoremap is written once, not re-read)
    const bool fuse_up = !tc_tuning().no_seg_fusion;
    if ((rc = run_handsegnet(ctx, image, B, H, W, fuse_up ? nullptr : seg, stream))) return rc;
    // single_obj_scoremap + calc_center_bb + scale (nets/...:82-85)
    int nl = 0;
    if ((rc = launch_seg_postprocess(seg, B, H, W, L.seg_scratch, hand_mask, nullptr, cen, L.crop_size, scl, s, &nl,
                                     fuse_up ? L.seg_low : nullptr, H / 8, W / 8))) return rc;
    ctx->launches += nl;
    if (force_center) H3D_CUDA(cudaMemcpyAsync(cen, force_center, (size_t)B * 8, cudaMemcpyDeviceToDevice, s));
    if (force_scale) H3D_CUDA(cudaMemcpyAsync(scl, force_scale, (size_t)B * 4, cudaMemcpyDeviceToDevice, s));
    // crop_image_from_xy (nets/...:86)
    if ((rc = launch_crop_image(image, cen, scl, crop, B, H, W, 3, 256, s))) return rc;
    ctx->launches += 1;
    // PoseNet2D (nets/...:89-90)
    if ((rc = h3d_posenet_forward(ctx, crop, B, 256, 256, nullptr, nullptr, nullptr, stream))) return rc;
    // x8 up-sampling (nets/...:96-97) and detect_keypoints (utils/general.py:331-344), fused when both are requested; it only
    // reads the 32x32 score map, so it runs on a side stream concurrently with the lifting stage
    const bool overlap = with_pose3d && !tc_tuning().no_side_stream;
    cudaStream_t us = s;
    if (overlap) {
        H3D_CUDA(cudaEventRecord(ctx->ev_fork2, s));
        H3D_CUDA(cudaStreamWaitEvent(ctx->side2, ctx->ev_fork2, 0));
        us = ctx->side2;
    }
    int rc_up;
    if (keypoints_uv) {
        nl = 0;
        rc_up = launch_resize_argmax21(L.s[2], kps, B, 32, 32, 256, 256, L.argmax_scratch, keypoints_uv, us, &nl);
        ctx->launches += nl;
    } else {
        rc_up = launch_resize_bilinear_tf1(L.s[2], kps, B, 32, 32, 21, 256, 256, us);
        ctx->launches += 1;
    }
    if (overlap) H3D_CUDA(cudaEventRecord(ctx->ev_join2, ctx->side2));
    if (rc_up) {   // never leave the side stream un-joined
        if (overlap) cudaStreamWaitEvent(s, ctx->ev_join2, 0);
        return rc_up;
    }
    // PosePrior + ViewpointNet on the 32x32 map (nets/...:93)
    if (with_pose3d)
        rc = h3d_lifting_forward(ctx, L.s[2], hand_side, B, H3D_VARIANT_PROPOSED, keypoint_coord3d, nullptr, nullptr, stream);
    if (overlap) H3D_CUDA(cudaStreamWaitEvent(s, ctx->ev_join2, 0));   // join even when the lifting stage failed
    if (rc) return rc;
    return H3D_OK;
}

// ---------------------------------------------------------------------------------------------- operators
// Every operator entry ENQUEUES only: scratch comes from the context (op_scratch), never from a per-call cudaMalloc, and nothing
// synchronises.  The one documented exception is h3d_conv2d_tc(_strided), which takes HOST weights and therefore packs, uploads and
// frees them around the call (test / tuning entry); its enqueue-only form is h3d_pack_conv_weights + h3d_conv2d_tc_packed.
#define H3D_OP_PROLOGUE(ctx)                              \
    H3D_REQUIRE((ctx) != nullptr, "ctx is NULL");         \
    DeviceGuard guard_((ctx)->device);                    \
    cudaStream_t s = (cudaStream_t)stream;

struct h3d_packed_conv { PackedW pw; int k = 0, Cin = 0, Cout = 0, precision = 0; };

int h3d_conv2d_f32(h3d_ctx* ctx, const float* x, const float* w_hwio, const float* bias, float* y, int B, int H, int W, int Cin,
                   int Cout, int ksize, int stride, int leaky, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    DirectConvArgs a;
    a.x = x; a.Cin_total = Cin; a.cin_off = 0; a.w = w_hwio; a.bias = bias; a.y = y; a.Cout_total = Cout; a.cout_off = 0;
    a.ys = Split(); a.Cs_total = 0; a.cs_off = 0; a.half = Half16::BF16;
    a.B = B; a.H = H; a.W = W; a.Cin = Cin; a.Cout = Cout; a.k = ksize; a.stride = stride; a.leaky = leaky;
    a.err_flag = ctx->err_flag;
    // lets tiny layers take the split-K path exactly as the lifting stage does
    const bool tiny = (int64_t)B * ceil_div(H, stride) * ceil_div(W, stride) <= 64 * 295;
    if (tiny) {
        char* scratch = nullptr;
        int rc0 = op_scratch(ctx, kConvSplitKScratchFloats * 4, &scratch);
        if (rc0) return rc0;
        a.splitk_scratch = (float*)scratch; a.splitk_scratch_floats = kConvSplitKScratchFloats;
    }
    int rc = launch_conv_direct(a, s);
    if (!rc) ctx->launches += conv_direct_num_launches(a);
    return rc;
}

int h3d_pack_conv_weights(h3d_ctx* ctx, const float* host_w_hwio, const float* host_bias, int ksize, int Cin, int Cout, int precision,
                          h3d_packed_conv** out) {
    H3D_REQUIRE(ctx && host_w_hwio && host_bias && out, "h3d_pack_conv_weights: NULL argument");
    H3D_REQUIRE(precision >= H3D_PREC_BF16X3 && precision <= H3D_PREC_FP16_F8C, "h3d_pack_conv_weights: precision must be a tensor-core mode");
    H3D_REQUIRE(ksize == 1 || ksize == 3 || ksize == 5 || ksize == 7, "h3d_pack_conv_weights: ksize must be 1, 3, 5 or 7");
    DeviceGuard guard(ctx->device);
    auto* h = new h3d_packed_conv();
    h->k = ksize; h->Cin = Cin; h->Cout = Cout; h->precision = precision;
    int rc = pack_conv_weights(host_w_hwio, host_bias, ksize, Cin, Cout, (int)align_up(Cin, 64), (int)align_up(Cout, 64), {}, half_of(precision),
                               passes_of(precision), &h->pw);
    if (rc) { free_packed(h->pw); delete h; return rc; }
    *out = h;
    return H3D_OK;
}

int h3d_free_packed_conv(h3d_ctx* ctx, h3d_packed_conv* packed) {
    if (!packed) return H3D_OK;
    H3D_REQUIRE(ctx != nullptr, "h3d_free_packed_conv: ctx is NULL");
    DeviceGuard guard(ctx->device);
    free_packed(packed->pw);     // cudaFree waits for kernels that still read the planes
    delete packed;
    return H3D_OK;
}

// Body shared by h3d_conv2d_tc_packed and h3d_conv2d_tc_dev.  Operand planes are carved from the context's operator scratch:
// [x hi | x lo / l8 h8 | y hi | y lo / l8 h8 | wbytes for the caller's weight planes]; pack(wbase, &pw) provides the packed weights
// (enqueueing their packing when they live in the scratch) before x is split and the convolution runs.
extern "C++" {   // a template inside the C ABI block
template <class PackFn>
static int conv_tc_run(h3d_ctx* ctx, const float* x, float* y, int B, int H, int W, int Cin, int Cout, int ksize, int stride, int leaky,
                       int precision, int Cin_pad, int Cout_pad, int64_t wbytes, PackFn pack, cudaStream_t s) {
    H3D_REQUIRE(stride == 1 || (stride == 2 && H % 2 == 0 && W % 2 == 0 && ksize >= 3),
                "h3d_conv2d_tc: stride must be 1, or 2 with even H and W and ksize >= 3 (for ksize 1 TF's 'SAME' samples the even pixels)");
    const Half16 half = half_of(precision);
    const int passes = passes_of(precision);
    const int64_t rows = (int64_t)B * H * W, rows_out = rows / (stride * stride);
    const int64_t xb = align_up(rows * Cin_pad * 2, 1024), yb = align_up(rows_out * Cout_pad * 2, 1024);
    char* base = nullptr;
    int rc = op_scratch(ctx, 2 * xb + 2 * yb + wbytes, &base);
    if (rc) return rc;
    PackedW pw;
    if ((rc = pack(base + 2 * xb + 2 * yb, &pw))) return rc;
    Split xs, ys;
    xs.hi = (uint16_t*)base; ys.hi = (uint16_t*)(base + 2 * xb);
    if (passes == 3) { xs.lo = (uint16_t*)(base + xb); ys.lo = (uint16_t*)(base + 2 * xb + yb); }
    if (passes == 4) {
        xs.l8 = (uint8_t*)(base + xb); xs.h8 = xs.l8 + align_up(rows * Cin_pad, 1024);
        ys.l8 = (uint8_t*)(base + 2 * xb + yb); ys.h8 = ys.l8 + align_up(rows_out * Cout_pad, 1024);
    }
    if ((rc = launch_f32_to_split(x, xs, rows, Cin, Cin_pad, half, s))) return rc;
    TcConvDesc d;
    d.x = xs; d.Cin_total = Cin_pad; d.Cin_pad = Cin_pad; d.w = pw.w; d.bias = pw.bias; d.w_scale = pw.w_scale; d.Cout = Cout;
    d.Cout_pad = Cout_pad;
    d.y = ys; d.Cy_total = Cout_pad; d.cy_off = 0; d.yf = nullptr; d.Cyf_total = 0; d.cyf_off = 0;
    d.B = B; d.H = H; d.W = W; d.k = ksize; d.leaky = leaky; d.passes = passes; d.half = half; d.corr_scale = pw.corr_scale;
    d.pool = stride == 2 ? 2 : 0;
    d.err_flag = ctx->err_flag;
    TcConvPlan* tp = tc_conv_plan_create(d);     // host-side only: tensor maps + launch geometry (passed to the kernel by value)
    if (!tp) return H3D_ECUDA;
    rc = tc_conv_launch(tp, s);
    tc_conv_plan_destroy(tp);
    if (rc) return rc;
    if ((rc = launch_split_to_f32(ys, y, rows_out, Cout, Cout_pad, half, s))) return rc;
    ctx->launches += 3;
    return H3D_OK;
}
}  // extern "C++"

int h3d_conv2d_tc_packed(h3d_ctx* ctx, const float* x, const h3d_packed_conv* packed, float* y, int B, int H, int W, int stride,
                         int leaky, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(x && packed && y && B > 0, "h3d_conv2d_tc_packed: bad argument");
    return conv_tc_run(ctx, x, y, B, H, W, packed->Cin, packed->Cout, packed->k, stride, leaky, packed->precision, packed->pw.Cin_pad,
                       packed->pw.Cout_pad, 0, [&](char*, PackedW* pw) { *pw = packed->pw; return (int)H3D_OK; }, s);
}

// Weight planes of a device-weight convolution in the operator scratch: [hi | lo | bias padded to Cout_pad | fp16: w_scale [Cout_pad]]
static int64_t dev_plane_bytes(int ksize, int Cin_pad, int Cout_pad) { return align_up((int64_t)Cout_pad * ksize * ksize * Cin_pad * 2, 1024); }

int h3d_conv2d_tc_dev(h3d_ctx* ctx, const float* x, const float* w_hwio, const float* bias, float* y, int B, int H, int W, int Cin,
                      int Cout, int ksize, int stride, int leaky, int precision, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(x && w_hwio && bias && y && B > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0, "h3d_conv2d_tc_dev: bad argument");
    H3D_REQUIRE(precision >= H3D_PREC_BF16X3 && precision <= H3D_PREC_BF16,
                "h3d_conv2d_tc_dev: precision must be bf16x3, fp16x3, fp16 or bf16 (fp16_f8c derives its scales from host weights)");
    H3D_REQUIRE(ksize == 1 || ksize == 3 || ksize == 5 || ksize == 7, "h3d_conv2d_tc_dev: ksize must be 1, 3, 5 or 7");
    const int Cin_pad = (int)align_up(Cin, 64), Cout_pad = (int)align_up(Cout, 64);
    const int64_t pb = dev_plane_bytes(ksize, Cin_pad, Cout_pad);
    auto pack = [&](char* wbase, PackedW* pw) {
        pw->w.hi = (uint16_t*)wbase;
        if (passes_of(precision) == 3) pw->w.lo = (uint16_t*)(wbase + pb);
        pw->bias = (float*)(wbase + 2 * pb);
        if (half_of(precision) == Half16::FP16) pw->w_scale = pw->bias + Cout_pad;
        pw->Cin_pad = Cin_pad; pw->Cout_pad = Cout_pad;
        ctx->launches += pw->w_scale ? 2 : 1;
        return launch_pack_conv_w(w_hwio, bias, pw->w, pw->bias, pw->w_scale, ksize, Cin, Cout, Cin_pad, Cout_pad, false, half_of(precision), s);
    };
    return conv_tc_run(ctx, x, y, B, H, W, Cin, Cout, ksize, stride, leaky, precision, Cin_pad, Cout_pad, 2 * pb + align_up(Cout_pad * 8, 1024),
                       pack, s);
}

int h3d_conv2d_tc_backward(h3d_ctx* ctx, const float* x, const float* y, const float* dy, const float* w_hwio, float* dx, float* dw_hwio,
                           float* db, int B, int H, int W, int Cin, int Cout, int ksize, int stride, int leaky, int precision, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(dy && B > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0, "h3d_conv2d_tc_backward: bad argument");
    H3D_REQUIRE(precision == H3D_PREC_BF16X3 || precision == H3D_PREC_BF16,
                "h3d_conv2d_tc_backward: precision must be bf16x3 or bf16 (fp16 planes have no range for small gradients without loss "
                "scaling, fp16_f8c carries per-layer scale factors, fp32_ffma has no tensor-core backward)");
    H3D_REQUIRE(ksize == 1 || ksize == 3 || ksize == 5 || ksize == 7, "h3d_conv2d_tc_backward: ksize must be 1, 3, 5 or 7");
    H3D_REQUIRE(stride == 1 || (stride == 2 && H % 2 == 0 && W % 2 == 0 && ksize >= 3),
                "h3d_conv2d_tc_backward: stride must be 1, or 2 with even H and W and ksize >= 3");
    H3D_REQUIRE(Cout <= 1024, "h3d_conv2d_tc_backward: Cout must be <= 1024");
    H3D_REQUIRE(!leaky || y, "h3d_conv2d_tc_backward: y (the forward output) is required with leaky");
    H3D_REQUIRE(!dx || w_hwio, "h3d_conv2d_tc_backward: dx needs w_hwio");
    H3D_REQUIRE(!dw_hwio || x, "h3d_conv2d_tc_backward: dw_hwio needs x");
    if (!dx && !dw_hwio && !db) return H3D_OK;
    const int passes = passes_of(precision);
    const int Cin_pad = (int)align_up(Cin, 64), Cout_pad = (int)align_up(Cout, 64);
    const int64_t rows = (int64_t)B * H * W;
    int64_t ppb = 0;
    const int nblk = conv_grad_prep_blocks(rows, &ppb);
    // scratch: [dy' hi | dy' lo | x hi | x lo | W_d hi | W_d lo | zero bias | db partials | dW partials]
    const int64_t gb = align_up(rows * Cout_pad * 2, 1024), xb = align_up(rows * Cin_pad * 2, 1024);
    const int64_t wb = dev_plane_bytes(ksize, Cin_pad, Cout_pad), zb = align_up(Cin_pad * 4, 1024);
    const int64_t dbb = align_up((int64_t)nblk * Cout_pad * 4, 1024);
    const int64_t pwb = dw_hwio ? conv_wgrad_partial_floats(B, H, W, ksize, Cin_pad, Cout_pad) * 4 : 0;
    char* base = nullptr;
    int rc = op_scratch(ctx, 2 * gb + 2 * xb + 2 * wb + zb + dbb + pwb, &base);
    if (rc) return rc;
    char* const xbase = base + 2 * gb;
    char* const wbase = xbase + 2 * xb;
    float* const zbias = (float*)(wbase + 2 * wb);
    float* const db_part = (float*)((char*)zbias + zb);
    float* const wpart = (float*)((char*)db_part + dbb);
    Split gs;
    gs.hi = (uint16_t*)base;
    if (passes == 3) gs.lo = (uint16_t*)(base + gb);
    if ((rc = launch_conv_grad_prep(dy, leaky ? y : nullptr, gs, db ? db_part : nullptr, B, H, W, Cout, Cout_pad, stride, leaky, s))) return rc;
    ctx->launches += 1;
    if (db) {
        if ((rc = launch_bias_grad_reduce(db_part, nblk, Cout, Cout_pad, db, s))) return rc;
        ctx->launches += 1;
    }
    if (dx) {   // the stride-1 'SAME' convolution of dy' with the flipped, transposed kernel, on the forward kernel
        Split wd;
        wd.hi = (uint16_t*)wbase;
        if (passes == 3) wd.lo = (uint16_t*)(wbase + wb);
        if ((rc = launch_pack_conv_w(w_hwio, nullptr, wd, zbias, nullptr, ksize, Cin, Cout, Cin_pad, Cout_pad, true, Half16::BF16, s))) return rc;
        TcConvDesc d;
        d.x = gs; d.Cin_total = Cout_pad; d.Cin_pad = Cout_pad; d.w = wd; d.bias = zbias; d.Cout = Cin; d.Cout_pad = Cin_pad;
        d.y = Split(); d.Cy_total = 0; d.cy_off = 0; d.yf = dx; d.Cyf_total = Cin; d.cyf_off = 0;
        d.B = B; d.H = H; d.W = W; d.k = ksize; d.leaky = 0; d.passes = passes; d.half = Half16::BF16; d.pool = 0;
        d.err_flag = ctx->err_flag;
        TcConvPlan* tp = tc_conv_plan_create(d);
        if (!tp) return H3D_ECUDA;
        rc = tc_conv_launch(tp, s);
        tc_conv_plan_destroy(tp);
        if (rc) return rc;
        ctx->launches += 2;
    }
    if (dw_hwio) {
        Split xs;
        xs.hi = (uint16_t*)xbase;
        if (passes == 3) xs.lo = (uint16_t*)(xbase + xb);
        if ((rc = launch_f32_to_split(x, xs, rows, Cin, Cin_pad, Half16::BF16, s))) return rc;
        WgradDesc d;
        d.x = xs; d.dy = gs;
        d.B = B; d.H = H; d.W = W; d.Cin = Cin; d.Cout = Cout; d.Cin_pad = Cin_pad; d.Cout_pad = Cout_pad; d.k = ksize; d.passes = passes;
        d.partial = wpart; d.dw = dw_hwio; d.err_flag = ctx->err_flag;
        if ((rc = launch_conv_wgrad(d, s))) return rc;
        ctx->launches += 3;
    }
    return H3D_OK;
}

int h3d_conv2d_tc(h3d_ctx* ctx, const float* x, const float* host_w_hwio, const float* host_bias, float* y, int B, int H, int W,
                  int Cin, int Cout, int ksize, int leaky, int precision, void* stream) {
    return h3d_conv2d_tc_strided(ctx, x, host_w_hwio, host_bias, y, B, H, W, Cin, Cout, ksize, 1, leaky, precision, stream);
}

int h3d_conv2d_tc_strided(h3d_ctx* ctx, const float* x, const float* host_w_hwio, const float* host_bias, float* y, int B, int H, int W,
                          int Cin, int Cout, int ksize, int stride, int leaky, int precision, void* stream) {
    H3D_REQUIRE(ctx != nullptr, "ctx is NULL");
    h3d_packed_conv* pk = nullptr;
    int rc = h3d_pack_conv_weights(ctx, host_w_hwio, host_bias, ksize, Cin, Cout, precision, &pk);
    if (rc) return rc;
    rc = h3d_conv2d_tc_packed(ctx, x, pk, y, B, H, W, stride, leaky, stream);
    h3d_free_packed_conv(ctx, pk);               // host-weight convenience entry: the free waits for the kernel (documented exception)
    return rc;
}

int h3d_maxpool2x2_f32(h3d_ctx* ctx, const float* x, float* y, int B, int H, int W, int C, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    int rc = launch_maxpool_f32(x, y, B, H, W, C, s);
    if (!rc) ctx->launches += 1;
    return rc;
}
int h3d_maxpool2x2_backward_f32(h3d_ctx* ctx, const float* x, const float* dy, float* dx, int B, int H, int W, int C, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(x && dy && dx && B > 0 && H > 0 && W > 0 && C > 0, "h3d_maxpool2x2_backward_f32: bad argument");
    int rc = launch_maxpool_backward_f32(x, dy, dx, B, H, W, C, s);
    if (!rc) ctx->launches += 1;
    return rc;
}
int h3d_fully_connected_f32(h3d_ctx* ctx, const float* x, const float* w, const float* bias, float* y, int B, int in_features,
                            int out_features, int leaky, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    char* scratch = nullptr;
    const int64_t scratch_floats = fc_scratch_floats(B, in_features, out_features);
    int rc = op_scratch(ctx, scratch_floats * 4, &scratch);
    if (rc) return rc;
    rc = launch_fc(x, w, bias, y, (float*)scratch, scratch_floats, B, in_features, out_features, leaky, in_features, s);
    if (!rc) ctx->launches += 2;
    return rc;
}
int h3d_leaky_relu_f32(h3d_ctx* ctx, const float* x, float* y, int64_t n, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(x && y && n > 0, "h3d_leaky_relu_f32: bad argument");
    int rc = launch_leaky_relu(x, y, n, s);
    if (!rc) ctx->launches += 1;
    return rc;
}
int h3d_resize_bilinear_tf1(h3d_ctx* ctx, const float* x, float* y, int B, int H, int W, int C, int out_h, int out_w, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    int rc = launch_resize_bilinear_tf1(x, y, B, H, W, C, out_h, out_w, s);
    if (!rc) ctx->launches += 1;
    return rc;
}
int h3d_avgpool8(h3d_ctx* ctx, const float* x, float* y, int B, int H, int W, int C, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    int rc = launch_avgpool8(x, y, B, H, W, C, s);
    if (!rc) ctx->launches += 1;
    return rc;
}
int h3d_seg_postprocess(h3d_ctx* ctx, const float* logits, int B, int H, int W, uint8_t* hand_mask, int32_t* max_loc, float* center,
                        float* crop_size, float* scale_crop, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(logits && center && scale_crop, "h3d_seg_postprocess: logits, center and scale_crop are required");
    char* scratch = nullptr;
    int rc = op_scratch(ctx, seg_scratch_bytes(B, H, W), &scratch);
    if (rc) return rc;
    int nl = 0;
    rc = launch_seg_postprocess(logits, B, H, W, scratch, hand_mask, max_loc, center, crop_size, scale_crop, s, &nl);
    ctx->launches += nl;
    return rc;
}
int h3d_calc_center_bb(h3d_ctx* ctx, const float* mask, int B, int H, int W, float* center, float* bb, float* crop_size, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(mask && center && B > 0 && H > 0 && W > 0, "h3d_calc_center_bb: bad argument");
    int rc = launch_mask_bbox(mask, B, H, W, center, bb, crop_size, s);
    if (!rc) ctx->launches += 1;
    return rc;
}
int h3d_crop_image_from_xy(h3d_ctx* ctx, const float* image, const float* center, const float* scale, float* image_crop, int B,
                           int H, int W, int C, int crop_size, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    int rc = launch_crop_image(image, center, scale, image_crop, B, H, W, C, crop_size, s);
    if (!rc) ctx->launches += 1;
    return rc;
}
int h3d_detect_keypoints(h3d_ctx* ctx, const float* scoremaps, int B, int H, int W, int C, int32_t* keypoints_uv, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    char* scratch = nullptr;
    int rc = op_scratch(ctx, argmax_scratch_bytes(B, C), &scratch);
    if (rc) return rc;
    int nl = 0;
    rc = launch_detect_keypoints(scoremaps, B, H, W, C, scratch, keypoints_uv, s, &nl);
    ctx->launches += nl;
    return rc;
}
int h3d_upsample_detect_keypoints(h3d_ctx* ctx, const float* scoremaps, int B, int H, int W, int out_h, int out_w, float* scoremaps_up,
                                  int32_t* keypoints_uv, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(scoremaps && scoremaps_up && keypoints_uv && B > 0, "h3d_upsample_detect_keypoints: bad argument");
    char* scratch = nullptr;
    int rc = op_scratch(ctx, argmax_scratch_bytes(B, 21), &scratch);
    if (rc) return rc;
    int nl = 0;
    rc = launch_resize_argmax21(scoremaps, scoremaps_up, B, H, W, out_h, out_w, scratch, keypoints_uv, s, &nl);
    ctx->launches += nl;
    return rc;
}
int h3d_pack_records(h3d_ctx* ctx, const float* coord3d, const int32_t* keypoints_uv, const float* center, const float* scale_crop, int B,
                     float* records, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(coord3d && keypoints_uv && center && scale_crop && records && B > 0, "h3d_pack_records: bad argument");
    int rc = launch_pack_records(coord3d, keypoints_uv, center, scale_crop, B, records, s);
    if (!rc) ctx->launches += 1;
    return rc;
}
int h3d_gather_records_p2p(h3d_ctx* ctx, const float* coord3d, const int32_t* keypoints_uv, const float* center, const float* scale_crop,
                           int B, int max_batch, const uint64_t* peer_buffers, const uint64_t* peer_signals, uint64_t multicast_ptr, int rank,
                           int world, uint32_t epoch, int64_t parity_stride_floats, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(coord3d && keypoints_uv && center && scale_crop && peer_buffers && peer_signals, "h3d_gather_records_p2p: NULL argument");
    H3D_REQUIRE(max_batch >= B && parity_stride_floats >= (int64_t)world * max_batch * 108, "h3d_gather_records_p2p: parity stride too small");
    int rc = launch_gather_records_p2p(coord3d, keypoints_uv, center, scale_crop, B, peer_buffers, peer_signals, multicast_ptr, rank,
                                       world, epoch, parity_stride_floats, max_batch, ctx->err_flag, s);
    if (!rc) ctx->launches += 1;
    return rc;
}
int h3d_decode_records(h3d_ctx* ctx, int dataset, const uint8_t* records, int B, int step, float* header, float* image, uint8_t* mask,
                       uint8_t* visibility, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(records && image && B > 0 && (step == 1 || step == 2 || step == 4), "h3d_decode_records: bad argument");
    int rc;
    if (dataset == H3D_DATASET_RHD) {
        const int hdr = 42 * 3 + 42 * 2 + 9;                           // 219 floats = 876 B, then 2 B padding
        rc = launch_decode_records(records, 410520, hdr, 878, 320, 320, step, 878 + 320 * 320 * 3, 42, header, image, mask, visibility, B, s);
    } else if (dataset == H3D_DATASET_STB) {
        const int hdr = 21 * 3 + 21 * 3;                               // 126 floats = 504 B
        rc = launch_decode_records(records, 922104, hdr, 504, 480, 640, step, -1, 0, header, image, nullptr, nullptr, B, s);
    } else {
        set_error("h3d_decode_records: unknown dataset %d", dataset);
        return H3D_EINVAL;
    }
    if (!rc) ctx->launches += 1;
    return rc;
}
int h3d_rhd_reader_items(h3d_ctx* ctx, const float* header, const uint8_t* hand_parts, const uint8_t* visibility, int B, int use_wrist_coord,
                         int hand_crop, int crop_size, float* keypoint_xyz21, float* keypoint_uv21, uint8_t* keypoint_vis21, float* hand_side,
                         float* keypoint_scale, float* keypoint_xyz21_normed, float* crop_center, float* crop_scale, float* cam_mat, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(header && hand_parts && visibility && hand_side && B > 0 && crop_size > 1, "h3d_rhd_reader_items: bad argument");
    int rc = launch_rhd_items(header, hand_parts, visibility, B, use_wrist_coord, hand_crop, crop_size, keypoint_xyz21, keypoint_uv21, keypoint_vis21,
                              hand_side, keypoint_scale, keypoint_xyz21_normed, crop_center, crop_scale, cam_mat, s);
    if (!rc) ctx->launches += 1;
    return rc;
}
int h3d_stb_reader_items(h3d_ctx* ctx, const float* header, int B, int use_wrist_coord, float* keypoint_xyz21, float* keypoint_uv21,
                         uint8_t* keypoint_vis21, float* keypoint_scale, float* keypoint_xyz21_normed, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(header && B > 0, "h3d_stb_reader_items: bad argument");
    int rc = launch_stb_items(header, B, use_wrist_coord, keypoint_xyz21, keypoint_uv21, keypoint_vis21, keypoint_scale, keypoint_xyz21_normed, s);
    if (!rc) ctx->launches += 1;
    return rc;
}
int h3d_gaussian_scoremap(h3d_ctx* ctx, const float* coords_hw, const uint8_t* valid, int B, int N, int H, int W, float sigma, float* scoremap,
                          void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(coords_hw && scoremap && B > 0 && H > 0 && W > 0 && sigma > 0.f, "h3d_gaussian_scoremap: bad argument");
    int rc = launch_gaussian_map(coords_hw, valid, B, N, H, W, sigma, scoremap, s);
    if (!rc) ctx->launches += 1;
    return rc;
}
int h3d_canonical_trafo(h3d_ctx* ctx, const float* coords_xyz, const uint8_t* cond_right, int B, float* coords_can, float* rot_mat,
                        float* rot_mat_inv, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(coords_xyz && B > 0, "h3d_canonical_trafo: bad argument");
    int rc = launch_canonical_trafo(coords_xyz, cond_right, B, coords_can, rot_mat, rot_mat_inv, s);
    if (!rc) ctx->launches += 1;
    return rc;
}
int h3d_eval_keypoint_dist(h3d_ctx* ctx, const float* gt, const uint8_t* vis, const float* pred, int n, int D, float* dist, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(gt && vis && pred && dist && n > 0 && D >= 1 && D <= 4, "h3d_eval_keypoint_dist: bad argument");
    int rc = launch_eval_dist(gt, vis, pred, n, D, dist, s);
    if (!rc) ctx->launches += 1;
    return rc;
}
int h3d_bone_rel_trafo_inv(h3d_ctx* ctx, const float* coords_rel, float* coords_xyz, int B, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(coords_rel && coords_xyz && B > 0, "h3d_bone_rel_trafo_inv: bad argument");
    int rc = launch_bone_rel_trafo_inv(coords_rel, coords_xyz, B, s);
    if (!rc) ctx->launches += 1;
    return rc;
}
int h3d_rotate_canonical(h3d_ctx* ctx, const float* coord_can, const float* uxyz, const float* hand_side, int B, float* rot_mat,
                         float* coord_out, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    int rc = launch_rotate_canonical(coord_can, uxyz, hand_side, B, rot_mat, coord_out, s);
    if (!rc) ctx->launches += 1;
    return rc;
}
int h3d_flip_right_hand(h3d_ctx* ctx, const float* coords_xyz, const uint8_t* cond_right, int B, float* out, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(coords_xyz && cond_right && out && B > 0, "h3d_flip_right_hand: bad argument");
    int rc = launch_flip_right_hand(coords_xyz, cond_right, B, out, s);
    if (!rc) ctx->launches += 1;
    return rc;
}

// ---------------------------------------------------------------------------------------------- training (train.cu)
int h3d_resize_bilinear_tf1_backward(h3d_ctx* ctx, const float* dy, float* dx, int B, int H, int W, int C, int out_h, int out_w,
                                     void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(dy && dx, "h3d_resize_bilinear_tf1_backward: dy and dx are required");
    H3D_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && out_h > 0 && out_w > 0,
                "h3d_resize_bilinear_tf1_backward: bad shape B=%d H=%d W=%d C=%d out=%dx%d", B, H, W, C, out_h, out_w);
    char* scratch = nullptr;
    int rc = op_scratch(ctx, std::max<int64_t>(4, resize_grad_scratch_floats(B, H, W, C, out_h, out_w) * 4), &scratch);
    if (rc) return rc;
    int nl = 0;
    rc = launch_resize_bilinear_tf1_grad(dy, dx, (float*)scratch, B, H, W, C, out_h, out_w, s, &nl);
    ctx->launches += nl;
    return rc;
}
int h3d_scoremap_loss_forward(h3d_ctx* ctx, const float* pred, const float* target, const float* vis, int B, int H, int W, float* loss,
                              float* rms, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(pred && target && vis && loss && rms, "h3d_scoremap_loss_forward: pred, target, vis, loss and rms are required");
    H3D_REQUIRE(B > 0 && H > 0 && W > 0 && (int64_t)H * W <= (1 << 30), "h3d_scoremap_loss_forward: bad shape B=%d H=%d W=%d", B, H, W);
    char* scratch = nullptr;
    int rc = op_scratch(ctx, scoremap_loss_scratch_floats(B, H, W) * 4, &scratch);
    if (rc) return rc;
    rc = launch_scoremap_loss(pred, target, vis, (float*)scratch, B, H, W, loss, rms, s);
    if (!rc) ctx->launches += 2;
    return rc;
}
int h3d_scoremap_loss_backward(h3d_ctx* ctx, const float* pred, const float* target, const float* vis, const float* rms,
                               const float* grad_loss, int B, int H, int W, float* dpred, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(pred && target && vis && rms && dpred, "h3d_scoremap_loss_backward: pred, target, vis, rms and dpred are required");
    H3D_REQUIRE(B > 0 && H > 0 && W > 0 && (int64_t)H * W <= (1 << 30), "h3d_scoremap_loss_backward: bad shape B=%d H=%d W=%d", B, H, W);
    int rc = launch_scoremap_loss_grad(pred, target, vis, rms, grad_loss, dpred, B, H, W, s);
    if (!rc) ctx->launches += 1;
    return rc;
}
int h3d_softmax_xent_forward(h3d_ctx* ctx, const float* logits, const float* labels, int64_t rows, float* loss, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(logits && labels && loss, "h3d_softmax_xent_forward: logits, labels and loss are required");
    H3D_REQUIRE(rows > 0, "h3d_softmax_xent_forward: rows must be positive, got %lld", (long long)rows);
    H3D_REQUIRE(((uintptr_t)logits | (uintptr_t)labels) % 8 == 0, "h3d_softmax_xent_forward: logits and labels must be 8-byte aligned");
    char* scratch = nullptr;
    int rc = op_scratch(ctx, softmax_xent_scratch_floats(rows) * 4, &scratch);
    if (rc) return rc;
    rc = launch_softmax_xent(logits, labels, (float*)scratch, rows, loss, s);
    if (!rc) ctx->launches += 2;
    return rc;
}
int h3d_softmax_xent_backward(h3d_ctx* ctx, const float* logits, const float* labels, const float* grad_loss, int64_t rows, float* dlogits,
                              void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(logits && labels && dlogits, "h3d_softmax_xent_backward: logits, labels and dlogits are required");
    H3D_REQUIRE(rows > 0, "h3d_softmax_xent_backward: rows must be positive, got %lld", (long long)rows);
    H3D_REQUIRE(((uintptr_t)logits | (uintptr_t)labels | (uintptr_t)dlogits) % 8 == 0,
                "h3d_softmax_xent_backward: logits, labels and dlogits must be 8-byte aligned");
    int rc = launch_softmax_xent_grad(logits, labels, grad_loss, dlogits, rows, s);
    if (!rc) ctx->launches += 1;
    return rc;
}
int h3d_adam_state_set(h3d_ctx* ctx, float* state, float lr, float beta1_power, float beta2_power, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(state && ((uintptr_t)state % 16) == 0, "h3d_adam_state_set: state must be a 16-byte aligned device pointer");
    int rc = launch_adam_state_set(state, 7, lr, beta1_power, beta2_power, s);
    if (!rc) ctx->launches += 1;
    return rc;
}
int h3d_adam_set_lr(h3d_ctx* ctx, float* state, float lr, void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(state && ((uintptr_t)state % 16) == 0, "h3d_adam_set_lr: state must be a 16-byte aligned device pointer");
    int rc = launch_adam_state_set(state, 1, lr, 0.f, 0.f, s);
    if (!rc) ctx->launches += 1;
    return rc;
}
int h3d_adam_step(h3d_ctx* ctx, const h3d_adam_tensor* table, int num_tensors, float* state, float beta1, float beta2, float epsilon,
                  void* stream) {
    H3D_OP_PROLOGUE(ctx);
    H3D_REQUIRE(table && state && ((uintptr_t)state % 16) == 0, "h3d_adam_step: table and a 16-byte aligned state are required");
    H3D_REQUIRE(beta1 >= 0.f && beta1 < 1.f && beta2 >= 0.f && beta2 < 1.f && epsilon >= 0.f,
                "h3d_adam_step: need 0 <= beta1, beta2 < 1 and epsilon >= 0");
    int rc = launch_adam_step(table, num_tensors, state, beta1, beta2, epsilon, s);
    if (!rc) ctx->launches += 1;
    return rc;
}

}  // extern "C"

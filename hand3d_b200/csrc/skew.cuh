// Schedule-skew hooks: delays at the synchronisation points of the tensor-core rings, the cluster handshakes, the programmatic
// dependent launches and the tickets, so that a test can force the interleavings the hardware only rarely picks.
//
// H3D_SKEW(site, iter) expands to nothing unless the translation unit is built with -DH3D_SKEW_BUILD (python -m hand3d_b200.build
// --skew, which writes libhand3d_b200_skew.so; the product library never contains a hook).  In the skew build a hook reads the
// per-site config below from a device global and sleeps (__nanosleep) when the calling thread has the site's role and the loop
// iteration `iter` is a multiple of the site's period.  A non-zero seed turns the delay into a pseudo-random one in [0, ns], hashed
// from (seed, CTA, warpgroup, site, iter).  The role and the hash are warp-uniform, so a hook never splits a warp.
//
// Hooks sit only beside synchronisation that already exists (mbarrier waits and arrivals, between wgmma commit and wait, around the
// named barriers, before cluster barriers and distributed-shared-memory reads, after griddepcontrol.launch_dependents, before ticket
// atomics).  A hook never sits inside arithmetic and never changes an arrival count, a parity or control flow: it only moves time.
// A delay is capped at kSkewMaxNs, so the few thousand hooks a CTA passes add milliseconds, far below the ~2 s bound of mbar_wait.
//
// The config is set through h3d_set_tuning with the keys skew_<site>_{ns,role,period,seed} and skew_reset (conv_wgmma.cu:
// tc_set_tuning); the product build rejects them as unknown keys.  The config is uploaded with a synchronous cudaMemcpyToSymbol to the
// current device only, outside the library's streams: set it between launches, with no kernel in flight, on the device that will run
// the kernels (the schedule-skew tests use one device and synchronise between cases).
#pragma once

namespace h3d {

enum SkewSite {
    SKEW_PRODUCER = 0,   // TMA producer: after a stage's empty wait, before its expect_tx
    SKEW_CONSUMER = 1,   // wgmma consumer: after a stage's full wait, before the wgmma that read it are issued
    SKEW_COMMIT = 2,     // between wgmma commit and wgmma wait (the stage release follows the wait)
    SKEW_EPILOGUE = 3,   // before the named barriers of the epilogue staging buffer / the wgrad fragment reduction
    SKEW_CLUSTER = 4,    // before a cluster barrier and before a read of a peer's shared memory
    SKEW_PDL_TAIL = 5,   // after griddepcontrol.launch_dependents: the dependent grid may start against a primary that has not stored
    SKEW_TICKET = 6,     // before a ticket atomic or a first-occurrence key's atomicMax
    SKEW_SITES = 7
};

// role of a site: which threads sleep
enum SkewRole {
    SKEW_ALL = 0,         // every thread of every CTA
    SKEW_WG0 = 1,         // warpgroup 0 (threads 0-127): the TMA producer of the warp-specialised kernels
    SKEW_WG1 = 2,         // warpgroup 1 (threads 128-255)
    SKEW_WG2 = 3,         // warpgroup 2 (threads 256-383)
    SKEW_EVEN_CTA = 4,    // CTAs with an even blockIdx.x
    SKEW_ODD_CTA = 5,     // CTAs with an odd blockIdx.x
    SKEW_LAST_RANK = 6,   // the last CTA of its cluster
    SKEW_RANK0 = 8        // SKEW_RANK0 + r: cluster rank r (a launch without clusters is rank 0 of a cluster of one)
};

constexpr unsigned kSkewMaxNs = 4000;   // cap of one delay

struct SkewSiteCfg { unsigned ns, role, period, seed; };
struct SkewCfg { SkewSiteCfg site[SKEW_SITES]; };

// skew build: host side of the config (conv_wgmma.cu).  Every translation unit with hooks keeps its own device copy and registers an
// uploader when the library loads; skew_set() updates the host config and runs every uploader.
int skew_register(int (*upload)(const SkewCfg&));
int skew_set(const char* key, int value);

}  // namespace h3d

#ifdef H3D_SKEW_BUILD

namespace h3d {
namespace {

__device__ SkewCfg g_skew_cfg;

__device__ __forceinline__ unsigned skew_hash(unsigned x) {
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}

__device__ __forceinline__ void skew_delay(int site, int iter) {
    const SkewSiteCfg c = g_skew_cfg.site[site];
    if (c.ns == 0u) return;
    if (c.period > 1u && (unsigned)iter % c.period != 0u) return;
    const unsigned wg = threadIdx.x >> 7;
    unsigned rank, nrank;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(nrank));
    bool on;
    switch (c.role) {
        case SKEW_ALL: on = true; break;
        case SKEW_WG0: on = wg == 0; break;
        case SKEW_WG1: on = wg == 1; break;
        case SKEW_WG2: on = wg == 2; break;
        case SKEW_EVEN_CTA: on = (blockIdx.x & 1u) == 0u; break;
        case SKEW_ODD_CTA: on = (blockIdx.x & 1u) == 1u; break;
        case SKEW_LAST_RANK: on = rank + 1u == nrank; break;
        default: on = c.role >= SKEW_RANK0 && rank == c.role - SKEW_RANK0; break;
    }
    if (!on) return;
    unsigned ns = c.ns;
    if (c.seed) ns = skew_hash(c.seed ^ skew_hash(blockIdx.x * 0x9E3779B9u ^ skew_hash(((unsigned)site << 24) ^ (wg << 20) ^ (unsigned)iter))) % (c.ns + 1u);
    if (ns) __nanosleep(ns);
}

int skew_upload(const SkewCfg& c) { return (int)cudaMemcpyToSymbol(g_skew_cfg, &c, sizeof(SkewCfg)); }
[[maybe_unused]] const int skew_registered = skew_register(skew_upload);

}  // namespace
}  // namespace h3d

#define H3D_SKEW(site, iter) ::h3d::skew_delay((site), (int)(iter))

#else

#define H3D_SKEW(...) ((void)0)

#endif

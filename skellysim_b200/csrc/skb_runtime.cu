// skb_runtime.cu -- host side of libskelly_b200.so: evaluator contexts, the plain kernel's launch planning, the C ABI
// declared in include/skelly_b200.h (the symmetric and cross kernels' host side: skb_sym.cu), and the reference-named
// C++ entry points kernels::stokeslet_direct_gpu_impl / kernels::stresslet_direct_gpu_impl (SkellySim
// include/kernels.hpp:17-20) so the library links in place of src/core/kernels.cu.
//
// No CPU fallback exists here: every path ends in a CUDA launch or an error code.
#include "pair_kernels.cuh"
#include "stream_kernels.cuh"
#include "skb_internal.hpp"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

namespace skb {

// ------------------------------------------------------------------------------------------------
// errors / bookkeeping
// ------------------------------------------------------------------------------------------------
static thread_local std::string g_last_error = "";
static std::atomic<long long> g_launches{0};
static std::atomic<long long> g_buffer_allocs{0};

int set_error(int code, const char *fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_last_error = buf;
    return code;
}
const char *last_error() { return g_last_error.c_str(); }
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
long long launch_count() { return g_launches.load(std::memory_order_relaxed); }

// ------------------------------------------------------------------------------------------------
// launch planning
// ------------------------------------------------------------------------------------------------
template <int KIND, int T, int MINB, bool EXCL = false>
static cudaError_t launch_variant(const PairArgs &a, dim3 grid, cudaStream_t st) {
    pair_sum_kernel<KIND, T, MINB, EXCL><<<grid, kCtaThreads, SmemLayout<KIND, T, EXCL>::total_bytes, st>>>(a);
    return cudaGetLastError();
}

template <int KIND, int T, int MINB, bool EXCL = false> static cudaError_t set_smem_variant() {
    return cudaFuncSetAttribute(pair_sum_kernel<KIND, T, MINB, EXCL>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                SmemLayout<KIND, T, EXCL>::total_bytes);
}

template <int KIND, int T, int MINB> static int occupancy_variant() {
    using L = SmemLayout<KIND, T>;
    int nb = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, pair_sum_kernel<KIND, T, MINB>, kCtaThreads, L::total_bytes) !=
        cudaSuccess)
        nb = 1;
    return nb < 1 ? 1 : nb;
}

// min-blocks-per-SM hints (register caps at 128 threads/CTA): T=1:8 (64)  T=2:6 (85)  T=4:4 (128)  T=8:2 (255)
#define SKB_DISPATCH_T(KIND, T, CALL)                                                                                 \
    switch (T) {                                                                                                      \
    case 1: CALL(KIND, 1, 8); break;                                                                                  \
    case 2: CALL(KIND, 2, 6); break;                                                                                  \
    case 4: CALL(KIND, 4, 4); break;                                                                                  \
    default: CALL(KIND, 8, 2); break;                                                                                 \
    }

// the gradient kinds' one configuration: 10 accumulators and 3 coordinates per target leave room for two targets per
// thread at four CTAs per SM (-Xptxas -v: 122 registers, no spills, no stack frame)
constexpr int kGradT = 2, kGradTIndex = 1, kGradMinB = 4;

DeviceInfo query_device(int dev) {
    DeviceInfo di;
    di.dev = dev;
    cudaDeviceProp p;
    cudaSetDevice(dev);
    cudaGetDeviceProperties(&p, dev);
    di.num_sms = p.multiProcessorCount;
    const int Ts[4] = {1, 2, 4, 8};
    for (int k = 0; k < 2; ++k)
        for (int ti = 0; ti < 4; ++ti) {
            int occ = 1;
#define OCC_CALL(KIND, T, MINB) occ = occupancy_variant<KIND, T, MINB>()
            if (k == 0) {
                SKB_DISPATCH_T(kStokeslet, Ts[ti], OCC_CALL)
            } else {
                SKB_DISPATCH_T(kStresslet, Ts[ti], OCC_CALL)
            }
#undef OCC_CALL
            di.occupancy[k][ti] = occ;
        }
    di.occupancy[kStokesletGrad][kGradTIndex] = occupancy_variant<kStokesletGrad, kGradT, kGradMinB>();
    di.occupancy[kStressletGrad][kGradTIndex] = occupancy_variant<kStressletGrad, kGradT, kGradMinB>();
    return di;
}

// Pick targets-per-thread T and the number of source splits S.
//   cost(T,S) ~ (CTAs on the busiest SM) x (source tiles per CTA) x T x penalty(T, resident chains)
// The busiest SM runs ceil(n_ctas / num_sms) CTAs; a CTA's time is proportional to the pairs it owns
// (T targets/thread x tiles) because the FP64 pipe is shared by the co-resident CTAs.
LaunchPlan plan_launch(const DeviceInfo &di, int kind, long long n_trg, int n_src_tiles, int force_T, int force_S) {
    LaunchPlan best;
    double best_cost = 1e300;
    const int Ts[4] = {1, 2, 4, 8};
    for (int ti = 0; ti < 4; ++ti) {
        const int T = Ts[ti];
        if (force_T > 0 && T != force_T)
            continue;
        const int occ = di.occupancy[kind][ti];
        const long long tile_t = (long long)kCtaThreads * T;
        const long long n_tiles_t = (n_trg + tile_t - 1) / tile_t;
        // efficiency of the inner loop vs T (LDS + loop overhead amortised over T pairs).  Stokeslet kernel rates on an
        // H100 SXM (700 W) at 96 000 x 102 400 (scripts/probe_perf.py): T=8 634, T=4 615, T=2 604, T=1 562 Gpairs/s;
        // with these penalties the planner's pick is within 2 % of the fastest forced (T, S) there, at 32 000 x 40 000
        // and at 3 000 x 2 500
        const double t_pen = (T == 1) ? 1.18 : (T == 2) ? 1.11 : (T == 4) ? 0.985 : 0.955;
        const int s_max = std::min(n_src_tiles, kMaxSplits);
        for (int S = 1; S <= s_max; ++S) {
            if (force_S > 0 && S != std::min(force_S, s_max))
                continue;
            const int per = (n_src_tiles + S - 1) / S;
            const int S_eff = (n_src_tiles + per - 1) / per;
            if (S_eff != S && force_S <= 0)
                continue; // duplicate of a smaller S
            const long long n_ctas = n_tiles_t * S_eff;
            const long long per_sm = (n_ctas + di.num_sms - 1) / di.num_sms;
            // CTAs beyond the resident limit run in later waves; same total either way
            const double resident = (double)std::min<long long>(per_sm, occ);
            // latency hiding: want >= ~12 independent pair chains per scheduler (1 warp/CTA/SMSP, T chains each)
            // (T <= 2 evaluates two sources per iteration: 2 T chains per warp, stokeslet_two_sources)
            const double chains = resident * (T <= 2 ? 2 * T : T);
            // (and CTA slots left empty on the busiest SM cost latency hiding too: a grid that half fills the CTA slots
            // runs slower than one that fills them)
            const double fill = std::min(1.0, (double)per_sm / (double)occ);
            const double lat_pen = (chains >= 12.0 ? 1.0 : (12.0 / chains) * 0.5 + 0.5) * (1.0 + 0.25 * (1.0 - fill));
            // fixed per-CTA cost (barrier init, target staging, partial write) in units of source tiles
            const double cta_overhead = 0.5;
            double cost = (double)per_sm * ((double)per + cta_overhead) * T * t_pen * lat_pen;
            // reduction cost of S partial slabs, in the same units (tiny, breaks ties toward small S)
            cost += 1e-3 * S_eff;
            if (cost < best_cost) {
                best_cost = cost;
                best.T = T;
                best.n_splits = S_eff;
                best.tiles_per_split = per;
                best.grid_x = (unsigned)n_tiles_t;
            }
        }
    }
    return best;
}

int launch_pair_sum(const DeviceInfo &di, int kind, const double *d_r_src, const double *d_f_packed, long long n_src,
                    long long n_src_pad, const double *d_r_trg, long long n_trg, double *d_partial,
                    const LaunchPlan &plan, cudaStream_t st, const int *d_src_fid, const int *d_trg_fid) {
    PairArgs a;
    a.src_fid = d_src_fid;
    a.trg_fid = d_trg_fid;
    a.r_src = d_r_src;
    a.f_src = d_f_packed;
    a.r_trg = d_r_trg;
    a.partial = d_partial;
    a.n_trg = n_trg;
    a.n_src = n_src;
    a.n_src_tiles = (int)((n_src + kSrcTile - 1) / kSrcTile);
    a.tiles_per_split = plan.tiles_per_split;
    (void)n_src_pad;
    dim3 grid(plan.grid_x, plan.n_splits, 1);
    cudaError_t e = cudaSuccess;
#define LAUNCH_CALL(KIND, T, MINB) e = launch_variant<KIND, T, MINB>(a, grid, st)
#define LAUNCH_CALL_EXCL(KIND, T, MINB) e = launch_variant<KIND, T, MINB, true>(a, grid, st)
    if (kind == kStokeslet && d_src_fid) { // fused self-exclusion variant (same-id pairs contribute 0)
        if (!d_trg_fid)
            return set_error(SKB_ERR_INVALID, "launch_pair_sum: exclusion ids without target ids");
        SKB_DISPATCH_T(kStokeslet, plan.T, LAUNCH_CALL_EXCL)
    } else if (kind == kStokeslet) {
        SKB_DISPATCH_T(kStokeslet, plan.T, LAUNCH_CALL)
    } else if (kind == kStokesletGrad || kind == kStressletGrad) {
        if (plan.T != kGradT)
            return set_error(SKB_ERR_INVALID, "launch_pair_sum: the gradient kinds run at T = %d (plan: %d)", kGradT,
                             plan.T);
        e = kind == kStokesletGrad ? launch_variant<kStokesletGrad, kGradT, kGradMinB>(a, grid, st)
                                   : launch_variant<kStressletGrad, kGradT, kGradMinB>(a, grid, st);
    } else {
        SKB_DISPATCH_T(kStresslet, plan.T, LAUNCH_CALL)
    }
#undef LAUNCH_CALL
#undef LAUNCH_CALL_EXCL
    if (e != cudaSuccess)
        return set_error(SKB_ERR_CUDA, "pair_sum_kernel launch failed: %s", cudaGetErrorString(e));
    count_launch(1);
    return SKB_OK;
}

int launch_reduce(const double *d_partial, double *d_u, long long n_trg, int n_splits, double scale, int accumulate,
                  cudaStream_t st, int width) {
    const long long n3 = width * n_trg;
    const int bs = 256;
    if (n_splits >= 4 * kReduceWideWarps && n3 <= 32LL * 4096) // few targets, many splits
        reduce_partials_wide_kernel<<<(unsigned)((n3 + 31) / 32), 32 * kReduceWideWarps, 0, st>>>(
            d_partial, d_u, n3, n_splits, scale, accumulate);
    else
        reduce_partials_kernel<<<(unsigned)((n3 + bs - 1) / bs), bs, 0, st>>>(d_partial, d_u, n3, n_splits, scale,
                                                                              accumulate);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess)
        return set_error(SKB_ERR_CUDA, "reduce_partials_kernel launch failed: %s", cudaGetErrorString(e));
    count_launch(1);
    return SKB_OK;
}

// ------------------------------------------------------------------------------------------------
// device buffers
// ------------------------------------------------------------------------------------------------
int DevBuf::ensure(size_t bytes) {
    if (bytes <= cap)
        return SKB_OK;
    *this = DevBuf(); // the old buffer goes before the new one is allocated
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&ptr, want);
    if (e != cudaSuccess) {
        ptr = nullptr;
        return set_error(SKB_ERR_ALLOC, "cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
    }
    cap = want;
    g_buffer_allocs.fetch_add(1, std::memory_order_relaxed);
    return SKB_OK;
}

int DevBuf::upload(const void *h, size_t bytes, cudaStream_t st) {
    if (bytes == 0)
        return SKB_OK;
    SKB_TRY(ensure(bytes));
    CUDA_TRY(cudaMemcpyAsync(ptr, h, bytes, cudaMemcpyHostToDevice, st));
    return SKB_OK;
}

// ------------------------------------------------------------------------------------------------
// pageable -> device upload through a pinned, multi-threaded staging ring
// ------------------------------------------------------------------------------------------------
namespace {
struct StagingRing {
    static constexpr int kBufs = 4;
    static constexpr size_t kChunk = 16u << 20;
    static constexpr int kMaxDev = 64;
    void *buf[kBufs] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t ev[kMaxDev][kBufs] = {}; // events belong to a device: one set per device that uploads
    bool ev_ok[kMaxDev] = {};
    bool ok = false;
    std::mutex mu;
    bool init(int dev) {
        if (dev < 0 || dev >= kMaxDev)
            return false;
        if (!ok) {
            for (int i = 0; i < kBufs; ++i)
                if (cudaMallocHost(&buf[i], kChunk) != cudaSuccess) {
                    (void)cudaGetLastError();
                    return false;
                }
            ok = true;
        }
        if (!ev_ok[dev]) {
            for (int i = 0; i < kBufs; ++i)
                if (cudaEventCreateWithFlags(&ev[dev][i], cudaEventDisableTiming) != cudaSuccess) {
                    (void)cudaGetLastError();
                    return false;
                }
            ev_ok[dev] = true;
        }
        return true;
    }
};
StagingRing g_ring; // pinned host memory is not tied to a device: one ring per process (uploads are serialised)
} // namespace

int upload_pageable(void *d_dst, const void *h_src, size_t bytes, cudaStream_t st) {
    if (bytes == 0)
        return SKB_OK;
    std::lock_guard<std::mutex> lock(g_ring.mu);
    int dev = -1;
    (void)cudaGetDevice(&dev); // the caller made the stream's device current
    if (bytes < (8u << 20) || !g_ring.init(dev)) { // small, or no pinned memory to be had: the driver's own staging
        cudaError_t e = cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, st);
        if (e != cudaSuccess)
            return set_error(SKB_ERR_CUDA, "cudaMemcpyAsync H2D (%zu bytes): %s", bytes, cudaGetErrorString(e));
        e = cudaStreamSynchronize(st);
        return e == cudaSuccess ? SKB_OK : set_error(SKB_ERR_CUDA, "H2D copy: %s", cudaGetErrorString(e));
    }
    const unsigned hw = std::thread::hardware_concurrency();
    const int n_thr = (int)std::max(1u, std::min(8u, hw ? hw / 2 : 4u));
    size_t done = 0;
    int k = 0;
    cudaError_t e = cudaSuccess;
    while (done < bytes && e == cudaSuccess) {
        const int b = k % StagingRing::kBufs;
        const size_t len = std::min(StagingRing::kChunk, bytes - done);
        if (k >= StagingRing::kBufs)
            e = cudaEventSynchronize(g_ring.ev[dev][b]); // the copy that last used this buffer has left it
        if (e != cudaSuccess)
            break;
        const char *src = (const char *)h_src + done;
        char *dst = (char *)g_ring.buf[b];
        const size_t piece = (len + n_thr - 1) / n_thr;
        std::vector<std::thread> th;
        for (int t = 1; t < n_thr; ++t) {
            const size_t o = std::min(len, (size_t)t * piece), l = std::min(piece, len - o);
            if (l)
                th.emplace_back([=] { std::memcpy(dst + o, src + o, l); });
        }
        std::memcpy(dst, src, std::min(piece, len));
        for (auto &t : th)
            t.join();
        e = cudaMemcpyAsync((char *)d_dst + done, dst, len, cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess)
            e = cudaEventRecord(g_ring.ev[dev][b], st);
        done += len;
        ++k;
    }
    if (e == cudaSuccess)
        e = cudaStreamSynchronize(st);
    if (e != cudaSuccess)
        return set_error(SKB_ERR_CUDA, "staged H2D copy (%zu bytes): %s", bytes, cudaGetErrorString(e));
    return SKB_OK;
}

} // namespace skb

using namespace skb;

// The launch attributes of every kernel that has them: the dynamic shared memory of the kernels that use more than the
// default 48 KB, and the max-shared carve-out of pair_sym_kernel, pair_cross_kernel and the background row streamer
// that runs beside them (an SM switches its shared-memory configuration only when idle, so a different preference would
// keep them from sharing it).  Setting an attribute also loads the kernel.  This runs where a device is first taken into
// use (skb_ctx and skb_dense creation), so that no kernel is loaded lazily in the middle of a matvec -- for instance
// while a group member on the same device spins on a flag.
int skb::prepare_device(int dev) {
    static std::mutex mu;
    static std::vector<bool> done;
    std::lock_guard<std::mutex> lock(mu);
    CUDA_TRY(cudaSetDevice(dev));
    if (dev < (int)done.size() && done[dev])
        return SKB_OK;
    int major = 0, minor = 0;
    CUDA_TRY(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    CUDA_TRY(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
    // sm_90a code runs on compute capability 9.0 only (arch-specific targets are not forward compatible)
    if (major != 9 || minor != 0)
        return set_error(SKB_ERR_NO_DEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", dev, major,
                         minor);
    for (int T : {1, 2, 4, 8}) {
#define SMEM_CALL(KIND, T, MINB) CUDA_TRY((set_smem_variant<KIND, T, MINB>()))
#define SMEM_CALL_EXCL(KIND, T, MINB) CUDA_TRY((set_smem_variant<KIND, T, MINB, true>()))
        SKB_DISPATCH_T(kStokeslet, T, SMEM_CALL)
        SKB_DISPATCH_T(kStokeslet, T, SMEM_CALL_EXCL)
        SKB_DISPATCH_T(kStresslet, T, SMEM_CALL)
#undef SMEM_CALL
#undef SMEM_CALL_EXCL
    }
    CUDA_TRY((set_smem_variant<kStokesletGrad, kGradT, kGradMinB>()));
    CUDA_TRY((set_smem_variant<kStressletGrad, kGradT, kGradMinB>()));
    SKB_TRY(prepare_sym_kernels());
    CUDA_TRY(cudaFuncSetAttribute(dense_stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kStreamSmemBytes));
    CUDA_TRY(cudaFuncSetAttribute(dense_stream_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                  cudaSharedmemCarveoutMaxShared));
    SKB_TRY(prepare_fiber_kernels());
    if (dev >= (int)done.size())
        done.resize(dev + 1);
    done[dev] = true;
    return SKB_OK;
}

// ------------------------------------------------------------------------------------------------
// context
// ------------------------------------------------------------------------------------------------
static int check_kind(int kind) {
    if (kind != SKB_STOKESLET && kind != SKB_STRESSLET)
        return set_error(SKB_ERR_INVALID, "unknown kernel kind %d", kind);
    return SKB_OK;
}

skb_ctx::~skb_ctx() {
    while (!devs.empty()) { // each device's buffers are freed with that device current
        if (devs.back().stream) // (an entry a failed create never reached owns nothing)
            cudaSetDevice(devs.back().info.dev);
        devs.pop_back();
    }
    if (nccl)
        nccl_group_destroy(nccl);
}

static int ctx_create_impl(const int *ids, int n, skb_ctx **out) {
    if (!out)
        return set_error(SKB_ERR_INVALID, "skb_ctx_create: out == NULL");
    *out = nullptr;
    int n_dev = 0;
    cudaError_t e = cudaGetDeviceCount(&n_dev);
    if (e != cudaSuccess || n_dev == 0)
        return set_error(SKB_ERR_NO_DEVICE, "no CUDA device available (%s); this library has no CPU fallback",
                         e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    if (n < 1 || n > n_dev)
        return set_error(SKB_ERR_INVALID, "skb_ctx_create: n_gpus=%d but %d device(s) visible", n, n_dev);
    std::unique_ptr<skb_ctx> ctx(new skb_ctx);
    if (const char *e = getenv("SKB_SYMMETRIC")) // default of skb_ctx_set_symmetric for contexts created from now on
        ctx->sym_mode = std::max(-1, std::min(1, atoi(e)));
    ctx->devs.resize(n);
    for (int g = 0; g < n; ++g) {
        DeviceState &d = ctx->devs[g];
        const int dev = ids ? ids[g] : g;
        if (dev < 0 || dev >= n_dev)
            return set_error(SKB_ERR_INVALID, "device id %d out of range", dev);
        SKB_TRY(prepare_device(dev));
        d.info = query_device(dev);
        CUDA_TRY(cudaStreamCreateWithFlags(d.stream.out(), cudaStreamNonBlocking));
        // (d.aux_stream is created on first use by the symmetric path: most contexts of a flow never need one, and a
        // device has a finite number of hardware queues for independent streams)
        CUDA_TRY(cudaEventCreateWithFlags(d.ev_fork.out(), cudaEventDisableTiming));
        CUDA_TRY(cudaEventCreateWithFlags(d.ev_join.out(), cudaEventDisableTiming));
        CUDA_TRY(cudaEventCreate(d.ev_t0.out()));
        CUDA_TRY(cudaEventCreate(d.ev_t1.out()));
        CUDA_TRY(cudaEventCreate(d.ev_k0.out()));
        CUDA_TRY(cudaEventCreate(d.ev_k1.out()));
        CUDA_TRY(cudaEventCreate(d.ev_s0.out()));
        CUDA_TRY(cudaEventCreate(d.ev_s1.out()));
    }
    if (n > 1)
        SKB_TRY(nccl_group_create(ctx->devs.size(), [&](int g) { return ctx->devs[g].info.dev; }, &ctx->nccl));
    *out = ctx.release();
    return SKB_OK;
}

extern "C" {

const char *skb_version(void) { return "skelly_b200 0.1.0 (sm_90a)"; }
const char *skb_last_error_string(void) { return last_error(); }
int64_t skb_launch_count(void) { return launch_count(); }
int64_t skb_buffer_alloc_count(void) { return g_buffer_allocs.load(std::memory_order_relaxed); }

int skb_device_count(int *n) {
    if (!n)
        return set_error(SKB_ERR_INVALID, "skb_device_count: NULL");
    int c = 0;
    cudaError_t e = cudaGetDeviceCount(&c);
    if (e != cudaSuccess) {
        *n = 0;
        return set_error(SKB_ERR_NO_DEVICE, "cudaGetDeviceCount: %s", cudaGetErrorString(e));
    }
    *n = c;
    return SKB_OK;
}

int skb_ctx_create(int n_gpus, skb_ctx **out) { return ctx_create_impl(nullptr, n_gpus, out); }
int skb_ctx_create_on(const int *device_ids, int n_gpus, skb_ctx **out) {
    if (!device_ids)
        return set_error(SKB_ERR_INVALID, "skb_ctx_create_on: device_ids == NULL");
    return ctx_create_impl(device_ids, n_gpus, out);
}

int skb_ctx_destroy(skb_ctx *ctx) {
    if (!ctx)
        return SKB_OK;
    for (auto &d : ctx->devs)
        if (d.stream)
            cudaStreamSynchronize(d.stream);
    delete ctx;
    return SKB_OK;
}

int skb_ctx_n_gpus(const skb_ctx *ctx, int *n) {
    if (!ctx || !n)
        return set_error(SKB_ERR_INVALID, "skb_ctx_n_gpus: NULL");
    *n = (int)ctx->devs.size();
    return SKB_OK;
}

int skb_ctx_set_tuning(skb_ctx *ctx, int T, int S) {
    if (!ctx)
        return set_error(SKB_ERR_INVALID, "skb_ctx_set_tuning: NULL ctx");
    if (!(T == 0 || T == 1 || T == 2 || T == 4 || T == 8) || S < 0)
        return set_error(SKB_ERR_INVALID, "tuning: targets_per_thread must be 0/1/2/4/8, source_splits >= 0");
    ctx->force_T = T;
    ctx->force_S = S;
    return SKB_OK;
}

int skb_ctx_set_symmetric(skb_ctx *ctx, int mode) {
    if (!ctx || mode < -1 || mode > 1)
        return set_error(SKB_ERR_INVALID, "skb_ctx_set_symmetric: mode must be -1 (auto), 0 (off) or 1 (on)");
    ctx->sym_mode = mode;
    return SKB_OK;
}

int skb_plan_query(int kind, int64_t n_trg, int64_t n_src, int num_sms, const int *occupancy4, int force_T,
                   int force_S, int *T, int *n_splits, int *tiles_per_split, int *grid_x) {
    if ((kind != 0 && kind != 1) || n_trg < 1 || n_src < 1 || num_sms < 1 || !occupancy4 || !T || !n_splits ||
        !tiles_per_split || !grid_x)
        return set_error(SKB_ERR_INVALID, "skb_plan_query: bad arguments");
    DeviceInfo di;
    di.num_sms = num_sms;
    for (int i = 0; i < 4; ++i)
        di.occupancy[kind][i] = std::max(1, occupancy4[i]);
    const LaunchPlan p = plan_launch(di, kind, n_trg, (int)((n_src + kSrcTile - 1) / kSrcTile), force_T, force_S);
    *T = p.T;
    *n_splits = p.n_splits;
    *tiles_per_split = p.tiles_per_split;
    *grid_x = (int)p.grid_x;
    return SKB_OK;
}

int skb_ctx_last_eval_was_symmetric(const skb_ctx *ctx, int *yes) {
    if (!ctx || !yes)
        return set_error(SKB_ERR_INVALID, "skb_ctx_last_eval_was_symmetric: NULL");
    *yes = ctx->last_was_sym ? 1 : 0;
    return SKB_OK;
}

int skb_ctx_set_sym_partition(skb_ctx *ctx, int part, int n_parts) {
    if (!ctx || n_parts < 1 || part < 0 || part >= n_parts)
        return set_error(SKB_ERR_INVALID, "skb_ctx_set_sym_partition: need 0 <= part < n_parts");
    if (ctx->devs.size() != 1)
        return set_error(SKB_ERR_INVALID, "skb_ctx_set_sym_partition: single-GPU contexts only");
    ctx->devs[0].sym_part = part;
    ctx->devs[0].sym_parts = n_parts;
    return SKB_OK;
}

int skb_last_eval_stats(const skb_ctx *ctx, skb_eval_stats *out) {
    if (!ctx || !out)
        return set_error(SKB_ERR_INVALID, "skb_last_eval_stats: NULL");
    *out = ctx->stats;
    if (ctx->kernel_events_pending) {
        // asynchronous evaluation: the events are valid once the caller's stream has passed them
        const DeviceState &d = ctx->devs[0];
        float ms = 0;
        cudaSetDevice(d.info.dev);
        if (cudaEventElapsedTime(&ms, d.ev_k0, d.ev_k1) == cudaSuccess)
            out->kernel_ms = ms;
        else
            (void)cudaGetLastError(); // not ready yet: leave 0
    }
    return SKB_OK;
}

} // extern "C"

// ------------------------------------------------------------------------------------------------
// positions
// ------------------------------------------------------------------------------------------------
static void partition_targets(skb_ctx *ctx, long long n_trg) {
    const long long P = (long long)ctx->devs.size();
    const long long chunk = (n_trg + P - 1) / P;
    for (long long g = 0; g < P; ++g) {
        DeviceState &d = ctx->devs[g];
        d.trg_begin = std::min(n_trg, g * chunk);
        d.n_trg = std::min(n_trg, (g + 1) * chunk) - d.trg_begin;
    }
    ctx->n_trg = n_trg;
}

static int set_targets_impl(skb_ctx *ctx, const double *r_trg, long long n_trg, bool on_device, cudaStream_t user) {
    // on_device: `user` is used verbatim (0 = CUDA's legacy default stream); host path: the context's stream
    if (!ctx)
        return set_error(SKB_ERR_INVALID, "set_targets: NULL ctx");
    if (n_trg < 0 || (n_trg > 0 && !r_trg))
        return set_error(SKB_ERR_INVALID, "set_targets: bad arguments (n_trg=%lld)", n_trg);
    if (on_device && ctx->devs.size() != 1)
        return set_error(SKB_ERR_INVALID, "device-pointer entry points need a single-GPU context");
    if (!on_device && ctx->devs.size() > 1) {
        // multi-device context: the device layout of the targets (plain block partition, or the symmetric layout
        // when they start with the Stokeslet sources) is decided at the next evaluation, see update_layout()
        ctx->h_trg.assign(r_trg, r_trg + 3 * n_trg);
        ctx->n_trg = n_trg;
        ctx->layout_dirty = true;
        return SKB_OK;
    }
    partition_targets(ctx, n_trg);
    for (auto &d : ctx->devs) {
        d.src[0].sym.self_state = -1;
        d.src[0].excl_trg_n = -1;
        if (d.n_trg == 0)
            continue;
        CUDA_TRY(cudaSetDevice(d.info.dev));
        SKB_TRY(d.r_trg.ensure((size_t)d.n_trg * 24));
        SKB_TRY(d.u.ensure((size_t)d.n_trg * 24));
        cudaStream_t st = on_device ? user : d.stream;
        CUDA_TRY(cudaMemcpyAsync(d.r_trg.ptr, r_trg + 3 * d.trg_begin, (size_t)d.n_trg * 24,
                                 on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
    }
    if (!on_device)
        for (auto &d : ctx->devs) {
            CUDA_TRY(cudaSetDevice(d.info.dev));
            CUDA_TRY(cudaStreamSynchronize(d.stream));
        }
    return SKB_OK;
}

// Multi-device contexts (host-pointer API): put the targets on the devices.  Plain layout: contiguous blocks.
// Symmetric layout (the targets start with the Stokeslet sources, no stresslet sources in this context): every
// device holds ALL n_self leading targets -- it evaluates its serpentine share of the self-interaction's block rows
// and produces partial sums for all of them -- followed by its block of the remaining targets.
static int update_layout(skb_ctx *ctx) {
    if (ctx->devs.size() < 2 || !ctx->layout_dirty)
        return SKB_OK;
    const long long P = (long long)ctx->devs.size();
    const long long n_trg = ctx->n_trg;
    const long long n_sl = ctx->devs[0].src[SKB_STOKESLET].n, n_dl = ctx->devs[0].src[SKB_STRESSLET].n;
    const long long block = sym_block_nodes();
    bool want = ctx->sym_mode != 0 && n_dl <= 0 && n_sl >= (ctx->sym_mode == 1 ? 2 * block : 4096) && n_trg >= n_sl &&
                (long long)ctx->h_src[SKB_STOKESLET].size() == 3 * n_sl &&
                std::memcmp(ctx->h_trg.data(), ctx->h_src[SKB_STOKESLET].data(), (size_t)n_sl * 24) == 0;
    if (want) {
        const long long n_pad = ctx->devs[0].src[SKB_STOKESLET].n_pad;
        if (((n_pad / block + P - 1) / P) * n_pad * 24 > sym_mem_budget())
            want = false;
    }
    ctx->sym_layout = want;
    ctx->n_self = want ? n_sl : 0;
    if (!want) {
        partition_targets(ctx, n_trg);
        for (auto &d : ctx->devs) {
            d.sym_part = 0;
            d.sym_parts = 1;
            d.rem_begin = d.rem_count = 0;
        }
    } else {
        const long long n_rem = n_trg - n_sl, chunk = (n_rem + P - 1) / P;
        for (long long g = 0; g < P; ++g) {
            DeviceState &d = ctx->devs[g];
            d.rem_begin = std::min(n_rem, g * chunk);
            d.rem_count = std::min(n_rem, (g + 1) * chunk) - d.rem_begin;
            d.trg_begin = 0;
            d.n_trg = n_sl + d.rem_count;
            d.sym_part = (int)g;
            d.sym_parts = (int)P;
        }
    }
    for (auto &d : ctx->devs) {
        d.src[0].sym.self_state = want ? 1 : 0; // decided on the host copies
        if (d.n_trg == 0)
            continue;
        CUDA_TRY(cudaSetDevice(d.info.dev));
        const long long chunk_f = want ? (ctx->n_self + P - 1) / P : 0;
        const long long u_rows = std::max(d.n_trg, chunk_f * P);
        SKB_TRY(d.r_trg.ensure((size_t)d.n_trg * 24));
        SKB_TRY(d.u.ensure((size_t)u_rows * 24));
        if (want) {
            SKB_TRY(d.u_rs.ensure((size_t)chunk_f * 24));
            CUDA_TRY(cudaMemcpyAsync(d.r_trg.ptr, ctx->h_trg.data(), (size_t)ctx->n_self * 24, cudaMemcpyHostToDevice,
                                     d.stream));
            if (d.rem_count > 0)
                CUDA_TRY(cudaMemcpyAsync((double *)d.r_trg.ptr + 3 * ctx->n_self,
                                         ctx->h_trg.data() + 3 * (ctx->n_self + d.rem_begin), (size_t)d.rem_count * 24,
                                         cudaMemcpyHostToDevice, d.stream));
        } else {
            CUDA_TRY(cudaMemcpyAsync(d.r_trg.ptr, ctx->h_trg.data() + 3 * d.trg_begin, (size_t)d.n_trg * 24,
                                     cudaMemcpyHostToDevice, d.stream));
        }
    }
    for (auto &d : ctx->devs) {
        CUDA_TRY(cudaSetDevice(d.info.dev));
        CUDA_TRY(cudaStreamSynchronize(d.stream));
    }
    ctx->layout_dirty = false;
    return SKB_OK;
}

static int set_sources_impl(skb_ctx *ctx, int kind, const double *r_src, long long n_src, bool on_device,
                            cudaStream_t user) {
    if (!ctx)
        return set_error(SKB_ERR_INVALID, "set_sources: NULL ctx");
    SKB_TRY(check_kind(kind));
    if (n_src < 0 || (n_src > 0 && !r_src))
        return set_error(SKB_ERR_INVALID, "set_sources: bad arguments (n_src=%lld)", n_src);
    if (n_src > (1LL << 31) - 1 - kSrcTile)
        return set_error(SKB_ERR_INVALID, "set_sources: n_src=%lld exceeds the supported range", n_src);
    if (on_device && ctx->devs.size() != 1)
        return set_error(SKB_ERR_INVALID, "device-pointer entry points need a single-GPU context");
    const long long kPadTo = 1024; // multiple of every source tile / symmetric block size in use
    const long long n_pad = ((n_src + kPadTo - 1) / kPadTo) * kPadTo;
    const int fdim_raw = kind == SKB_STOKESLET ? 3 : 9;
    const int fdim_packed = kind == SKB_STOKESLET ? 3 : 6;
    const long long P = (long long)ctx->devs.size();
    const long long chunk = (n_src + P - 1) / P; // all-gather slot per device
    if (!on_device && P > 1) {
        ctx->h_src[kind].assign(r_src, r_src + 3 * n_src);
        ctx->layout_dirty = true;
    }
    for (auto &d : ctx->devs) {
        SourceSet &s = d.src[kind];
        s.n = n_src;
        s.n_pad = n_pad;
        s.has_normals = false;
        s.has_weights = false;
        s.excl = false;    // ids belong to one set of sources
        s.excl_trg_n = -1;
        s.sym.self_state = -1; // (the symmetric plan depends on the block count only and survives position updates)
        if (n_src == 0)
            continue;
        CUDA_TRY(cudaSetDevice(d.info.dev));
        cudaStream_t st = on_device ? user : d.stream;
        SKB_TRY(s.r.ensure((size_t)n_pad * 24));
        SKB_TRY(s.f_raw.ensure((size_t)chunk * P * fdim_raw * 8));
        SKB_TRY(s.f_packed.ensure((size_t)n_pad * fdim_packed * 8));
        const double *d_in = r_src;
        if (!on_device) {
            SKB_TRY(d.scratch.ensure((size_t)n_src * 24));
            CUDA_TRY(cudaMemcpyAsync(d.scratch.ptr, r_src, (size_t)n_src * 24, cudaMemcpyHostToDevice, st));
            d_in = (const double *)d.scratch.ptr;
        }
        const int bs = 256;
        pad_positions_kernel<<<(unsigned)((n_pad * 3 + bs - 1) / bs), bs, 0, st>>>(d_in, (double *)s.r.ptr, n_src,
                                                                                   n_pad);
        CUDA_TRY(cudaGetLastError());
        count_launch(1);
    }
    if (!on_device)
        for (auto &d : ctx->devs) {
            CUDA_TRY(cudaSetDevice(d.info.dev));
            CUDA_TRY(cudaStreamSynchronize(d.stream));
        }
    return SKB_OK;
}

// ------------------------------------------------------------------------------------------------
// evaluation
// ------------------------------------------------------------------------------------------------
namespace skb {
__global__ void excl_target_ids_kernel(const int *__restrict__ src_ids, long long n_src, long long trg_begin,
                                       long long n_trg, int *__restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_trg) {
        const long long g = trg_begin + i; // global target row: the leading n_src rows are the sources themselves
        out[i] = g < n_src ? src_ids[g] : -1;
    }
}

int pack_on_device(DeviceState &d, int kind, StrengthMode mode, const double *d_f_raw, double two_eta, cudaStream_t st,
                   int *launches) {
    SourceSet &s = d.src[kind];
    const int bs = 256;
    s.f_cur = (const double *)s.f_packed.ptr;
    if (s.n <= 0)
        return SKB_OK;
    if (kind == SKB_STOKESLET) {
        pack_sl_kernel<<<(unsigned)((s.n_pad * 3 + bs - 1) / bs), bs, 0, st>>>(
            d_f_raw, s.has_weights ? (const double *)s.weights.ptr : nullptr, (double *)s.f_packed.ptr, s.n, s.n_pad);
    } else if (mode == kRaw) {
        pack_dl9_kernel<<<(unsigned)((s.n_pad + bs - 1) / bs), bs, 0, st>>>(d_f_raw, (double *)s.f_packed.ptr, s.n,
                                                                             s.n_pad);
    } else {
        pack_dl_normal_density_kernel<<<(unsigned)((s.n_pad + bs - 1) / bs), bs, 0, st>>>(
            (const double *)s.normals.ptr, d_f_raw, two_eta, (double *)s.f_packed.ptr, s.n, s.n_pad);
    }
    CUDA_TRY(cudaGetLastError());
    count_launch(1);
    if (launches)
        *launches += 1;
    return SKB_OK;
}

int eval_on_device(skb_ctx *ctx, DeviceState &d, int kind, StrengthMode mode, const double *d_f_raw, double two_eta,
                   double *d_u_out, int accumulate, cudaStream_t st, bool record_events, int *launches,
                   LaunchPlan *plan_out, double scale_mul, const EvalOpts &opts) {
    SourceSet &s = d.src[kind];
    const int bs = 256;
    if (d.n_trg == 0)
        return SKB_OK;
    if (s.n == 0) {
        if (!accumulate)
            CUDA_TRY(cudaMemsetAsync(d_u_out, 0, (size_t)d.n_trg * 24, st));
        return SKB_OK;
    }
    // 1. strengths -> packed, padded layout
    if (mode == kPacked)
        s.f_cur = d_f_raw;
    else
        SKB_TRY(pack_on_device(d, kind, mode, d_f_raw, two_eta, st, launches));
    if (record_events)
        CUDA_TRY(cudaEventRecord(d.ev_k0, st));
    // fused self-exclusion (opt-in): ids only make sense when the sources are the leading targets
    const bool excl = kind == SKB_STOKESLET && s.excl;
    if (excl && ctx->devs.size() == 1) { // (multi-device contexts check their host copies of the positions, eval_host)
        SKB_TRY(ensure_self_state(d, s, st));
        if (s.sym.self_state != 1)
            return set_error(SKB_ERR_STATE, "exclusion ids are set, but the targets do not start with the Stokeslet "
                                            "sources (skb_set_source_exclusion_ids)");
    }
    // 2. pair sums
    // ---- symmetric path: sources are the leading targets (fiber -> fiber block of apply_matvec) ----
    long long n_sym = 0;
    if (kind == SKB_STOKESLET && (ctx->devs.size() == 1 || ctx->sym_layout) && ctx->sym_mode != 0) {
        int use = 0;
        SKB_TRY(sym_prepare(ctx, d, st, &use));
        if (use)
            n_sym = s.n;
    }
    const long long n_trg_std = d.n_trg - n_sym; // targets beyond the square block go through the plain kernel
    const double *d_r_trg_std = (const double *)d.r_trg.ptr + 3 * n_sym;
    double *d_u_std = (n_sym > 0 && opts.d_u_rem) ? opts.d_u_rem : d_u_out + 3 * n_sym;
    const double scale = scale_mul * (kind == SKB_STOKESLET ? 1.0 : -3.0) / (8.0 * M_PI);
    cudaStream_t st_std = st;
    if (n_sym > 0 && !d.aux_stream)
        CUDA_TRY(cudaStreamCreateWithFlags(d.aux_stream.out(), cudaStreamNonBlocking));
    if (n_sym > 0 && n_trg_std > 0) { // fork: the remainder fills the SMs the symmetric kernel's tail leaves idle
        CUDA_TRY(cudaEventRecord(d.ev_fork, st));
        CUDA_TRY(cudaStreamWaitEvent(d.aux_stream, d.ev_fork, 0));
        st_std = d.aux_stream;
    }
    LaunchPlan plan{};
    // the long symmetric kernel is launched first so that the remainder's CTAs are dispatched into its tail
    if (n_sym > 0)
        SKB_TRY(sym_eval(d, opts.d_u_sym ? opts.d_u_sym : d_u_out,
                         opts.sym_accumulate >= 0 ? opts.sym_accumulate : accumulate, st, scale_mul, launches));
    if (n_trg_std > 0) {
        const int *d_src_ids = nullptr, *d_trg_ids = nullptr;
        if (excl && n_sym == 0) { // the whole target list goes through the plain kernel: it needs per-target ids
            if (s.excl_trg_n != d.n_trg) {
                SKB_TRY(s.excl_trg.ensure((size_t)d.n_trg * sizeof(int)));
                excl_target_ids_kernel<<<(unsigned)((d.n_trg + bs - 1) / bs), bs, 0, st_std>>>(
                    (const int *)s.excl_ids.ptr, s.n, d.trg_begin, d.n_trg, (int *)s.excl_trg.ptr);
                CUDA_TRY(cudaGetLastError());
                count_launch(1);
                s.excl_trg_n = d.n_trg;
            }
            d_src_ids = (const int *)s.excl_ids.ptr;
            d_trg_ids = (const int *)s.excl_trg.ptr;
        } // (with the symmetric path the remainder targets are not sources: nothing to exclude there)
        plan = plan_launch(d.info, kind, n_trg_std, (int)((s.n + kSrcTile - 1) / kSrcTile), ctx->force_T, ctx->force_S);
        SKB_TRY(d.partial.ensure((size_t)plan.n_splits * (size_t)n_trg_std * 24));
        SKB_TRY(launch_pair_sum(d.info, kind, (const double *)s.r.ptr, s.f_cur, s.n, s.n_pad, d_r_trg_std, n_trg_std,
                                (double *)d.partial.ptr, plan, st_std, d_src_ids, d_trg_ids));
        // 3. combine splits, scale: 1/(8 pi) (kernels.cu:59) or -3/(8 pi) (kernels.cu:26,51)
        SKB_TRY(launch_reduce((const double *)d.partial.ptr, d_u_std, n_trg_std, plan.n_splits, scale, accumulate,
                              st_std));
        if (launches)
            *launches += 2;
    }
    if (kind == SKB_STOKESLET)
        ctx->last_was_sym = n_sym > 0;
    if (n_sym > 0) {
        if (n_trg_std > 0) { // join
            CUDA_TRY(cudaEventRecord(d.ev_join, d.aux_stream));
            CUDA_TRY(cudaStreamWaitEvent(st, d.ev_join, 0));
        }
        plan = sym_launch_plan(s);
    }
    if (record_events)
        CUDA_TRY(cudaEventRecord(d.ev_k1, st));
    if (plan_out)
        *plan_out = plan;
    return SKB_OK;
}

int eval_gradient_on_device(DeviceState &d, int kind, StrengthMode mode, const double *d_f_raw, double two_eta,
                            double *d_g, cudaStream_t st, int *launches, double scale_mul) {
    SourceSet &s = d.src[kind];
    if (d.n_trg == 0 || s.n <= 0)
        return SKB_OK;
    SKB_TRY(pack_on_device(d, kind, mode, d_f_raw, two_eta, st, launches));
    const int gkind = kind == SKB_STOKESLET ? kStokesletGrad : kStressletGrad;
    constexpr int kOut = KindTraits<kStokesletGrad>::odim;
    const LaunchPlan plan = plan_launch(d.info, gkind, d.n_trg, (int)((s.n + kSrcTile - 1) / kSrcTile), kGradT, 0);
    SKB_TRY(d.partial.ensure((size_t)plan.n_splits * (size_t)d.n_trg * kOut * 8));
    SKB_TRY(launch_pair_sum(d.info, gkind, (const double *)s.r.ptr, s.f_cur, s.n, s.n_pad, (const double *)d.r_trg.ptr,
                            d.n_trg, (double *)d.partial.ptr, plan, st));
    const double scale = scale_mul * (kind == SKB_STOKESLET ? 1.0 : -3.0) / (8.0 * M_PI);
    SKB_TRY(launch_reduce((const double *)d.partial.ptr, d_g, d.n_trg, plan.n_splits, scale, 1, st, kOut));
    if (launches)
        *launches += 2;
    return SKB_OK;
}
} // namespace skb

// host-pointer evaluation over all devices of the context
static int eval_host(skb_ctx *ctx, int kind, StrengthMode mode, const double *f_src, double eta, double *u_trg,
                     int accumulate) {
    if (!ctx)
        return set_error(SKB_ERR_INVALID, "eval: NULL ctx");
    SKB_TRY(check_kind(kind));
    if (ctx->n_trg < 0)
        return set_error(SKB_ERR_STATE, "eval: skb_set_targets has not been called");
    const long long n_src = ctx->devs[0].src[kind].n;
    if (n_src < 0)
        return set_error(SKB_ERR_STATE, "eval: skb_set_sources(kind=%d) has not been called", kind);
    if ((n_src > 0 && !f_src) || (ctx->n_trg > 0 && !u_trg))
        return set_error(SKB_ERR_INVALID, "eval: NULL strength or output pointer");
    if (mode == kNormalDensity && n_src > 0 && !ctx->devs[0].src[kind].has_normals)
        return set_error(SKB_ERR_STATE, "eval_double_layer: skb_set_source_normals has not been called");
    SKB_TRY(update_layout(ctx));
    if (kind == SKB_STOKESLET && ctx->devs.size() > 1 && ctx->devs[0].src[kind].excl &&
        !(ctx->n_trg >= n_src && (long long)ctx->h_src[kind].size() == 3 * n_src &&
          std::memcmp(ctx->h_trg.data(), ctx->h_src[kind].data(), (size_t)n_src * 24) == 0))
        return set_error(SKB_ERR_STATE, "exclusion ids are set, but the targets do not start with the Stokeslet sources "
                                        "(skb_set_source_exclusion_ids)");
    if (n_src == 0) { // an empty class contributes nothing, whatever layout the devices hold the targets in
        if (!accumulate && ctx->n_trg > 0)
            std::memset(u_trg, 0, (size_t)ctx->n_trg * 24);
        ctx->stats = skb_eval_stats{};
        return SKB_OK;
    }
    const bool sym_layout = ctx->sym_layout && kind == SKB_STOKESLET; // (no stresslet sources exist in that layout)
    const long long n_self = sym_layout ? ctx->n_self : 0;
    const int fdim = (kind == SKB_STOKESLET || mode == kNormalDensity) ? 3 : 9;
    const long long P = (long long)ctx->devs.size();
    const long long chunk = (n_src + P - 1) / P;
    int launches = 0;
    LaunchPlan plan{};

    // stage 1: strengths to the devices.  P == 1: one H2D.  P > 1: each device receives its 1/P slice over
    // PCIe, then ONE NCCL all-gather per evaluation distributes the slices over NVLink.
    for (long long g = 0; g < P; ++g) {
        DeviceState &d = ctx->devs[g];
        CUDA_TRY(cudaSetDevice(d.info.dev));
        CUDA_TRY(cudaEventRecord(d.ev_t0, d.stream));
        if (n_src == 0)
            continue;
        SourceSet &s = d.src[kind];
        const long long b = std::min(n_src, g * chunk), e = std::min(n_src, (g + 1) * chunk);
        if (e > b)
            CUDA_TRY(cudaMemcpyAsync((double *)s.f_raw.ptr + (size_t)g * chunk * fdim, f_src + (size_t)b * fdim,
                                     (size_t)(e - b) * fdim * 8, cudaMemcpyHostToDevice, d.stream));
    }
    if (P > 1 && n_src > 0) {
        std::vector<void *> bufs(P);
        std::vector<cudaStream_t> sts(P);
        for (long long g = 0; g < P; ++g) {
            bufs[g] = ctx->devs[g].src[kind].f_raw.ptr;
            sts[g] = ctx->devs[g].stream;
        }
        SKB_TRY(nccl_group_allgather_inplace(ctx->nccl, bufs.data(), (size_t)chunk * fdim, sts.data()));
    }
    // stage 2: every device evaluates its targets against all sources
    const long long chunk_f = sym_layout ? (n_self + P - 1) / P : 0; // reduce-scatter slot (leading rows per device)
    for (long long g = 0; g < P; ++g) {
        DeviceState &d = ctx->devs[g];
        if (d.n_trg == 0)
            continue;
        CUDA_TRY(cudaSetDevice(d.info.dev));
        if (!sym_layout) {
            if (accumulate)
                CUDA_TRY(cudaMemcpyAsync(d.u.ptr, u_trg + 3 * d.trg_begin, (size_t)d.n_trg * 24,
                                         cudaMemcpyHostToDevice, d.stream));
        } else {
            // leading rows are partial sums over the devices: the caller's values enter once (device 0)
            if (chunk_f * P > n_self)
                CUDA_TRY(cudaMemsetAsync((double *)d.u.ptr + 3 * n_self, 0, (size_t)(chunk_f * P - n_self) * 24,
                                         d.stream));
            if (accumulate) {
                if (g == 0)
                    CUDA_TRY(cudaMemcpyAsync(d.u.ptr, u_trg, (size_t)n_self * 24, cudaMemcpyHostToDevice, d.stream));
                else
                    CUDA_TRY(cudaMemsetAsync(d.u.ptr, 0, (size_t)n_self * 24, d.stream));
                if (d.rem_count > 0)
                    CUDA_TRY(cudaMemcpyAsync((double *)d.u.ptr + 3 * n_self, u_trg + 3 * (n_self + d.rem_begin),
                                             (size_t)d.rem_count * 24, cudaMemcpyHostToDevice, d.stream));
            }
        }
        SKB_TRY(eval_on_device(ctx, d, kind, mode, (const double *)d.src[kind].f_raw.ptr, 2.0 * eta,
                               (double *)d.u.ptr, accumulate, d.stream, true, &launches, g == 0 ? &plan : nullptr, 1.0));
        if (!sym_layout) {
            CUDA_TRY(cudaMemcpyAsync(u_trg + 3 * d.trg_begin, d.u.ptr, (size_t)d.n_trg * 24, cudaMemcpyDeviceToHost,
                                     d.stream));
            CUDA_TRY(cudaEventRecord(d.ev_t1, d.stream));
        }
    }
    if (sym_layout) {
        // one reduce-scatter of the leading rows: device g ends up with rows [g*chunk_f, (g+1)*chunk_f)
        std::vector<void *> send(P), recv(P);
        std::vector<cudaStream_t> sts(P);
        for (long long g = 0; g < P; ++g) {
            send[g] = ctx->devs[g].u.ptr;
            recv[g] = ctx->devs[g].u_rs.ptr;
            sts[g] = ctx->devs[g].stream;
        }
        SKB_TRY(nccl_group_reduce_scatter(ctx->nccl, send.data(), recv.data(), (size_t)chunk_f * 3, sts.data()));
        for (long long g = 0; g < P; ++g) {
            DeviceState &d = ctx->devs[g];
            CUDA_TRY(cudaSetDevice(d.info.dev));
            const long long b = std::min(n_self, g * chunk_f), e = std::min(n_self, (g + 1) * chunk_f);
            if (e > b)
                CUDA_TRY(cudaMemcpyAsync(u_trg + 3 * b, d.u_rs.ptr, (size_t)(e - b) * 24, cudaMemcpyDeviceToHost,
                                         d.stream));
            if (d.rem_count > 0)
                CUDA_TRY(cudaMemcpyAsync(u_trg + 3 * (n_self + d.rem_begin), (double *)d.u.ptr + 3 * n_self,
                                         (size_t)d.rem_count * 24, cudaMemcpyDeviceToHost, d.stream));
            CUDA_TRY(cudaEventRecord(d.ev_t1, d.stream));
        }
    }
    // stage 3: wait, collect timings
    double k_ms = 0, t_ms = 0;
    for (long long g = 0; g < P; ++g) {
        DeviceState &d = ctx->devs[g];
        CUDA_TRY(cudaSetDevice(d.info.dev));
        CUDA_TRY(cudaStreamSynchronize(d.stream));
        if (d.n_trg == 0)
            continue;
        float ms = 0;
        if (n_src > 0 && cudaEventElapsedTime(&ms, d.ev_k0, d.ev_k1) == cudaSuccess)
            k_ms = std::max(k_ms, (double)ms);
        if (cudaEventElapsedTime(&ms, d.ev_t0, d.ev_t1) == cudaSuccess)
            t_ms = std::max(t_ms, (double)ms);
    }
    ctx->kernel_events_pending = false;
    ctx->stats.kernel_ms = k_ms;
    ctx->stats.total_ms = t_ms;
    ctx->stats.n_pairs = n_src * ctx->n_trg;
    ctx->stats.launches = launches;
    ctx->stats.targets_per_thread = plan.T;
    ctx->stats.source_splits = plan.n_splits;
    ctx->stats.grid_ctas = (int)(plan.grid_x * plan.n_splits);
    return SKB_OK;
}

// process-wide context behind the stateless reference-shaped entry points
static std::mutex g_default_mu;
static skb_ctx *g_default_ctx = nullptr;
static int default_ctx(skb_ctx **out) {
    if (!g_default_ctx) {
        int rc = skb_ctx_create(1, &g_default_ctx);
        if (rc != SKB_OK)
            return rc;
    }
    *out = g_default_ctx;
    return SKB_OK;
}

static int direct_impl(int kind, const double *r_src, const double *f_src, int n_src, const double *r_trg,
                       double *u_trg, int n_trg) {
    if (n_src < 0 || n_trg < 0)
        return set_error(SKB_ERR_INVALID, "negative count");
    std::lock_guard<std::mutex> lock(g_default_mu);
    skb_ctx *ctx = nullptr;
    SKB_TRY(default_ctx(&ctx));
    SKB_TRY(skb_set_sources(ctx, kind, r_src, n_src));
    SKB_TRY(skb_set_targets(ctx, r_trg, n_trg));
    return skb_eval(ctx, kind, f_src, u_trg, 0);
}

extern "C" {

int skb_set_targets(skb_ctx *ctx, const double *r_trg, int64_t n_trg) {
    return set_targets_impl(ctx, r_trg, n_trg, false, nullptr);
}
int skb_set_targets_device(skb_ctx *ctx, const double *d_r_trg, int64_t n_trg, void *stream) {
    return set_targets_impl(ctx, d_r_trg, n_trg, true, (cudaStream_t)stream);
}
int skb_set_sources(skb_ctx *ctx, int kind, const double *r_src, int64_t n_src) {
    return set_sources_impl(ctx, kind, r_src, n_src, false, nullptr);
}
int skb_set_sources_device(skb_ctx *ctx, int kind, const double *d_r_src, int64_t n_src, void *stream) {
    return set_sources_impl(ctx, kind, d_r_src, n_src, true, (cudaStream_t)stream);
}

int skb_set_source_normals(skb_ctx *ctx, const double *normals, int64_t n_src) {
    if (!ctx)
        return set_error(SKB_ERR_INVALID, "set_source_normals: NULL ctx");
    const long long n = ctx->devs[0].src[SKB_STRESSLET].n;
    if (n < 0)
        return set_error(SKB_ERR_STATE, "set_source_normals: call skb_set_sources(SKB_STRESSLET, ...) first");
    if (n_src != n || (n > 0 && !normals))
        return set_error(SKB_ERR_INVALID, "set_source_normals: n_src=%lld does not match the %lld stresslet sources",
                         (long long)n_src, n);
    for (auto &d : ctx->devs) {
        SourceSet &s = d.src[SKB_STRESSLET];
        s.has_normals = true;
        if (n == 0)
            continue;
        CUDA_TRY(cudaSetDevice(d.info.dev));
        SKB_TRY(s.normals.ensure((size_t)n * 24));
        CUDA_TRY(cudaMemcpyAsync(s.normals.ptr, normals, (size_t)n * 24, cudaMemcpyHostToDevice, d.stream));
        CUDA_TRY(cudaStreamSynchronize(d.stream));
    }
    return SKB_OK;
}

int skb_set_source_exclusion_ids(skb_ctx *ctx, const int32_t *ids, int64_t n_src) {
    if (!ctx)
        return set_error(SKB_ERR_INVALID, "skb_set_source_exclusion_ids: NULL ctx");
    const long long n = ctx->devs[0].src[SKB_STOKESLET].n;
    if (n < 0)
        return set_error(SKB_ERR_STATE, "skb_set_source_exclusion_ids: call skb_set_sources(SKB_STOKESLET, ...) first");
    if (ids && n_src != n)
        return set_error(SKB_ERR_INVALID, "skb_set_source_exclusion_ids: n_src=%lld does not match the %lld Stokeslet "
                                          "sources", (long long)n_src, n);
    for (auto &d : ctx->devs) {
        SourceSet &s = d.src[SKB_STOKESLET];
        s.excl = false;
        s.excl_trg_n = -1;
        if (!ids || n == 0)
            continue;
        CUDA_TRY(cudaSetDevice(d.info.dev));
        SKB_TRY(s.excl_ids.ensure((size_t)s.n_pad * sizeof(int)));
        CUDA_TRY(cudaMemsetAsync(s.excl_ids.ptr, 0xff, (size_t)s.n_pad * sizeof(int), d.stream)); // pads: id -1
        CUDA_TRY(cudaMemcpyAsync(s.excl_ids.ptr, ids, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, d.stream));
        CUDA_TRY(cudaStreamSynchronize(d.stream));
        s.excl = true;
    }
    return SKB_OK;
}

int skb_eval(skb_ctx *ctx, int kind, const double *f_src, double *u_trg, int accumulate) {
    return eval_host(ctx, kind, kRaw, f_src, 0.0, u_trg, accumulate);
}

int skb_eval_double_layer(skb_ctx *ctx, const double *density, double eta, double *u_trg, int accumulate) {
    return eval_host(ctx, SKB_STRESSLET, kNormalDensity, density, eta, u_trg, accumulate);
}

int skb_eval_fused(skb_ctx *ctx, const double *f_sl, const double *f_dl, double *u_trg) {
    if (!ctx)
        return set_error(SKB_ERR_INVALID, "eval_fused: NULL ctx");
    int acc = 0;
    skb_eval_stats total{};
    if (f_sl) {
        SKB_TRY(eval_host(ctx, SKB_STOKESLET, kRaw, f_sl, 0.0, u_trg, acc));
        acc = 1;
        total = ctx->stats;
    }
    if (f_dl) {
        SKB_TRY(eval_host(ctx, SKB_STRESSLET, kRaw, f_dl, 0.0, u_trg, acc));
        acc = 1;
        total.kernel_ms += ctx->stats.kernel_ms;
        total.total_ms += ctx->stats.total_ms;
        total.n_pairs += ctx->stats.n_pairs;
        total.launches += ctx->stats.launches;
        total.targets_per_thread = ctx->stats.targets_per_thread;
        total.source_splits = ctx->stats.source_splits;
        total.grid_ctas = ctx->stats.grid_ctas;
        ctx->stats = total;
    }
    if (!acc && ctx->n_trg > 0) {
        if (!u_trg)
            return set_error(SKB_ERR_INVALID, "eval_fused: NULL output");
        std::memset(u_trg, 0, (size_t)ctx->n_trg * 24);
    }
    return SKB_OK;
}

int skb_eval_device(skb_ctx *ctx, int kind, const double *d_f_src, double *d_u_trg, int accumulate, void *stream) {
    if (!ctx)
        return set_error(SKB_ERR_INVALID, "eval_device: NULL ctx");
    SKB_TRY(check_kind(kind));
    if (ctx->devs.size() != 1)
        return set_error(SKB_ERR_INVALID, "device-pointer entry points need a single-GPU context");
    DeviceState &d = ctx->devs[0];
    if (ctx->n_trg < 0 || d.src[kind].n < 0)
        return set_error(SKB_ERR_STATE, "eval_device: targets / sources not set");
    if ((d.src[kind].n > 0 && !d_f_src) || (ctx->n_trg > 0 && !d_u_trg))
        return set_error(SKB_ERR_INVALID, "eval_device: NULL pointer");
    CUDA_TRY(cudaSetDevice(d.info.dev));
    cudaStream_t st = (cudaStream_t)stream; // verbatim: 0 is CUDA's legacy default stream
    int launches = 0;
    LaunchPlan plan{};
    SKB_TRY(eval_on_device(ctx, d, kind, kRaw, d_f_src, 0.0, d_u_trg, accumulate, st, true, &launches, &plan, 1.0));
    ctx->kernel_events_pending = d.src[kind].n > 0 && d.n_trg > 0;
    ctx->stats.kernel_ms = 0;
    ctx->stats.total_ms = 0;
    ctx->stats.n_pairs = d.src[kind].n * ctx->n_trg;
    ctx->stats.launches = launches;
    ctx->stats.targets_per_thread = plan.T;
    ctx->stats.source_splits = plan.n_splits;
    ctx->stats.grid_ctas = (int)(plan.grid_x * plan.n_splits);
    return SKB_OK;
}

int skb_sync(skb_ctx *ctx) {
    if (!ctx)
        return set_error(SKB_ERR_INVALID, "skb_sync: NULL ctx");
    for (auto &d : ctx->devs) {
        CUDA_TRY(cudaSetDevice(d.info.dev));
        CUDA_TRY(cudaStreamSynchronize(d.stream));
    }
    return SKB_OK;
}

int skb_stokeslet_direct(const double *r_src, const double *f_src, int n_src, const double *r_trg, double *u_trg,
                         int n_trg) {
    return direct_impl(SKB_STOKESLET, r_src, f_src, n_src, r_trg, u_trg, n_trg);
}
int skb_stresslet_direct(const double *r_src, const double *f_src, int n_src, const double *r_trg, double *u_trg,
                         int n_trg) {
    return direct_impl(SKB_STRESSLET, r_src, f_src, n_src, r_trg, u_trg, n_trg);
}

int skb_measure_fp64_peak(skb_ctx *ctx, double *flops_per_s) {
    if (!ctx || !flops_per_s)
        return set_error(SKB_ERR_INVALID, "skb_measure_fp64_peak: NULL");
    DeviceState &d = ctx->devs[0];
    CUDA_TRY(cudaSetDevice(d.info.dev));
    const int blocks = d.info.num_sms * 8, threads = 256, iters = 1 << 15;
    SKB_TRY(d.scratch.ensure((size_t)blocks * threads * 8));
    double best = 0;
    for (int rep = 0; rep < 5; ++rep) {
        CUDA_TRY(cudaEventRecord(d.ev_k0, d.stream));
        dfma_probe_kernel<<<blocks, threads, 0, d.stream>>>((double *)d.scratch.ptr, iters, 0.999999, 1e-9);
        CUDA_TRY(cudaGetLastError());
        count_launch(1);
        CUDA_TRY(cudaEventRecord(d.ev_k1, d.stream));
        CUDA_TRY(cudaStreamSynchronize(d.stream));
        float ms = 0;
        CUDA_TRY(cudaEventElapsedTime(&ms, d.ev_k0, d.ev_k1));
        const double fl = 2.0 * 8.0 * (double)iters * blocks * threads / (ms * 1e-3);
        if (rep > 0)
            best = std::max(best, fl);
    }
    *flops_per_s = best;
    return SKB_OK;
}

} // extern "C"

// ------------------------------------------------------------------------------------------------
// Reference-named C++ entry points (SkellySim include/kernels.hpp:17-20).  Linking this library in
// place of src/core/kernels.cu keeps kernels::stokeslet_direct_gpu / stresslet_direct_gpu
// (src/core/kernels.cpp:354-366) and `pair_evaluator = "GPU"` working unchanged.  Error behaviour
// follows the reference's CUDA path: message on stderr, exit(EXIT_FAILURE) (kernels.cu:8-15).
// ------------------------------------------------------------------------------------------------
namespace kernels {
__attribute__((visibility("default"))) void stokeslet_direct_gpu_impl(const double *r_src, const double *f_src,
                                                                      int n_src, const double *r_trg, double *u_trg,
                                                                      int n_trg) {
    if (skb_stokeslet_direct(r_src, f_src, n_src, r_trg, u_trg, n_trg) != SKB_OK) {
        fprintf(stderr, "skelly_b200: stokeslet_direct_gpu_impl: %s\n", skb_last_error_string());
        exit(EXIT_FAILURE);
    }
}
__attribute__((visibility("default"))) void stresslet_direct_gpu_impl(const double *r_src, const double *f_src,
                                                                      int n_src, const double *r_trg, double *u_trg,
                                                                      int n_trg) {
    if (skb_stresslet_direct(r_src, f_src, n_src, r_trg, u_trg, n_trg) != SKB_OK) {
        fprintf(stderr, "skelly_b200: stresslet_direct_gpu_impl: %s\n", skb_last_error_string());
        exit(EXIT_FAILURE);
    }
}
} // namespace kernels

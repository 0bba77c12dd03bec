// skb_runtime.cu -- the library-wide host side of libskelly_b200.so: errors and counters, device buffers, the staging
// ring, prepare_device, the plain kernel's launch planning, and the one-device Evaluator that flows and contexts
// evaluate through (its symmetric path: skb_sym.cu).  The evaluator contexts and their C ABI are skb_ctx.cu.
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
// use (flow, context and skb_dense creation), so that no kernel is loaded lazily in the middle of a matvec -- for instance
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

} // extern "C"

// ------------------------------------------------------------------------------------------------
// the evaluator of one device
// ------------------------------------------------------------------------------------------------
int skb::check_kind(int kind) {
    if (kind != SKB_STOKESLET && kind != SKB_STRESSLET)
        return set_error(SKB_ERR_INVALID, "unknown kernel kind %d", kind);
    return SKB_OK;
}

int skb::check_sources(int kind, const double *r, long long n) {
    SKB_TRY(check_kind(kind));
    if (n < 0 || (n > 0 && !r))
        return set_error(SKB_ERR_INVALID, "set_sources: bad arguments (n_src=%lld)", n);
    if (n > (1LL << 31) - 1 - kSrcTile)
        return set_error(SKB_ERR_INVALID, "set_sources: n_src=%lld exceeds the supported range", n);
    return SKB_OK;
}

int skb::launch_fp64_probe(double *d_out, int blocks, int threads, int iters, cudaStream_t st) {
    dfma_probe_kernel<<<blocks, threads, 0, st>>>(d_out, iters, 0.999999, 1e-9);
    CUDA_TRY(cudaGetLastError());
    count_launch(1);
    return SKB_OK;
}

namespace skb {
__global__ void excl_target_ids_kernel(const int *__restrict__ src_ids, long long n_src, long long trg_begin,
                                       long long n_trg, int *__restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_trg) {
        const long long g = trg_begin + i; // global target row: the leading n_src rows are the sources themselves
        out[i] = g < n_src ? src_ids[g] : -1;
    }
}

int Evaluator::init(const DeviceInfo &di) {
    info = di;
    if (const char *e = getenv("SKB_SYMMETRIC")) // default of sym_mode for evaluators made from now on
        sym_mode = std::max(-1, std::min(1, atoi(e)));
    // (aux_stream is created on first use by the symmetric path: most evaluators of a flow never need one, and a
    // device has a finite number of hardware queues for independent streams)
    CUDA_TRY(cudaEventCreateWithFlags(ev_fork.out(), cudaEventDisableTiming));
    CUDA_TRY(cudaEventCreateWithFlags(ev_join.out(), cudaEventDisableTiming));
    CUDA_TRY(cudaEventCreate(ev_s0.out()));
    CUDA_TRY(cudaEventCreate(ev_s1.out()));
    return SKB_OK;
}

int Evaluator::set_targets(const double *r, long long n, bool on_device, cudaStream_t st) {
    trg_begin = 0;
    n_trg = n;
    src[SKB_STOKESLET].sym.self_state = -1;
    src[SKB_STOKESLET].excl_trg_n = -1;
    if (n == 0)
        return SKB_OK;
    CUDA_TRY(cudaSetDevice(info.dev));
    SKB_TRY(r_trg.ensure((size_t)n * 24));
    CUDA_TRY(cudaMemcpyAsync(r_trg.ptr, r, (size_t)n * 24, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice,
                             st));
    return SKB_OK;
}

int Evaluator::set_sources(int kind, const double *r, long long n, bool on_device, cudaStream_t st, long long n_parts) {
    SKB_TRY(check_sources(kind, r, n));
    const long long kPadTo = 1024; // multiple of every source tile / symmetric block size in use
    const long long n_pad = ((n + kPadTo - 1) / kPadTo) * kPadTo;
    const int fdim_raw = kind == SKB_STOKESLET ? 3 : 9;
    const int fdim_packed = kind == SKB_STOKESLET ? 3 : 6;
    const long long chunk = (n + n_parts - 1) / n_parts; // all-gather slot per device
    SourceSet &s = src[kind];
    s.n = n;
    s.n_pad = n_pad;
    s.has_normals = false;
    s.has_weights = false;
    s.excl = false;    // ids belong to one set of sources
    s.excl_trg_n = -1;
    s.sym.self_state = -1; // (the symmetric plan depends on the block count only and survives position updates)
    if (n == 0)
        return SKB_OK;
    CUDA_TRY(cudaSetDevice(info.dev));
    SKB_TRY(s.r.ensure((size_t)n_pad * 24));
    SKB_TRY(s.f_raw.ensure((size_t)chunk * n_parts * fdim_raw * 8));
    SKB_TRY(s.f_packed.ensure((size_t)n_pad * fdim_packed * 8));
    const double *d_in = r;
    if (!on_device) {
        SKB_TRY(scratch.ensure((size_t)n * 24));
        CUDA_TRY(cudaMemcpyAsync(scratch.ptr, r, (size_t)n * 24, cudaMemcpyHostToDevice, st));
        d_in = (const double *)scratch.ptr;
    }
    const int bs = 256;
    pad_positions_kernel<<<(unsigned)((n_pad * 3 + bs - 1) / bs), bs, 0, st>>>(d_in, (double *)s.r.ptr, n, n_pad);
    CUDA_TRY(cudaGetLastError());
    count_launch(1);
    return SKB_OK;
}

int Evaluator::set_normals(const double *normals, long long n_src, cudaStream_t st) {
    SourceSet &s = src[SKB_STRESSLET];
    const long long n = s.n;
    if (n < 0)
        return set_error(SKB_ERR_STATE, "set_source_normals: call skb_set_sources(SKB_STRESSLET, ...) first");
    if (n_src != n || (n > 0 && !normals))
        return set_error(SKB_ERR_INVALID, "set_source_normals: n_src=%lld does not match the %lld stresslet sources",
                         n_src, n);
    s.has_normals = true;
    if (n == 0)
        return SKB_OK;
    CUDA_TRY(cudaSetDevice(info.dev));
    SKB_TRY(s.normals.ensure((size_t)n * 24));
    CUDA_TRY(cudaMemcpyAsync(s.normals.ptr, normals, (size_t)n * 24, cudaMemcpyHostToDevice, st));
    return SKB_OK;
}

int Evaluator::set_exclusion_ids(const int32_t *ids, long long n_src, cudaStream_t st) {
    SourceSet &s = src[SKB_STOKESLET];
    const long long n = s.n;
    if (n < 0)
        return set_error(SKB_ERR_STATE, "skb_set_source_exclusion_ids: call skb_set_sources(SKB_STOKESLET, ...) first");
    if (ids && n_src != n)
        return set_error(SKB_ERR_INVALID, "skb_set_source_exclusion_ids: n_src=%lld does not match the %lld Stokeslet "
                                          "sources", n_src, n);
    s.excl = false;
    s.excl_trg_n = -1;
    if (!ids || n == 0)
        return SKB_OK;
    CUDA_TRY(cudaSetDevice(info.dev));
    SKB_TRY(s.excl_ids.ensure((size_t)s.n_pad * sizeof(int)));
    CUDA_TRY(cudaMemsetAsync(s.excl_ids.ptr, 0xff, (size_t)s.n_pad * sizeof(int), st)); // pads: id -1
    CUDA_TRY(cudaMemcpyAsync(s.excl_ids.ptr, ids, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
    s.excl = true;
    return SKB_OK;
}

int Evaluator::pack(int kind, StrengthMode mode, const double *d_f_raw, double two_eta, cudaStream_t st,
                    int *launches) {
    SourceSet &s = src[kind];
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
    return launched(launches);
}

int Evaluator::eval(int kind, StrengthMode mode, const double *d_f_raw, double two_eta, double *d_u_out,
                    int accumulate, cudaStream_t st, int *launches, LaunchPlan *plan_out, double scale_mul,
                    const EvalOpts &opts, cudaEvent_t ev_k0, cudaEvent_t ev_k1) {
    SourceSet &s = src[kind];
    const int bs = 256;
    if (n_trg == 0)
        return SKB_OK;
    if (s.n == 0) {
        if (!accumulate)
            CUDA_TRY(cudaMemsetAsync(d_u_out, 0, (size_t)n_trg * 24, st));
        return SKB_OK;
    }
    // 1. strengths -> packed, padded layout
    if (mode == kPacked)
        s.f_cur = d_f_raw;
    else
        SKB_TRY(pack(kind, mode, d_f_raw, two_eta, st, launches));
    if (ev_k0)
        CUDA_TRY(cudaEventRecord(ev_k0, st));
    // fused self-exclusion (opt-in): ids only make sense when the sources are the leading targets
    const bool excl = kind == SKB_STOKESLET && s.excl;
    if (excl && layout != kBlocks) { // (the plain block layout's context checks its host copies of the positions)
        SKB_TRY(ensure_self_state(*this, s, st));
        if (s.sym.self_state != 1)
            return set_error(SKB_ERR_STATE, "exclusion ids are set, but the targets do not start with the Stokeslet "
                                            "sources (skb_set_source_exclusion_ids)");
    }
    // 2. pair sums
    // ---- symmetric path: sources are the leading targets (fiber -> fiber block of apply_matvec) ----
    long long n_sym = 0;
    if (kind == SKB_STOKESLET && layout != kBlocks && sym_mode != 0) {
        int use = 0;
        SKB_TRY(sym_prepare(*this, st, &use));
        if (use)
            n_sym = s.n;
    }
    const long long n_trg_std = n_trg - n_sym; // targets beyond the square block go through the plain kernel
    const double *d_r_trg_std = (const double *)r_trg.ptr + 3 * n_sym;
    double *d_u_std = (n_sym > 0 && opts.d_u_rem) ? opts.d_u_rem : d_u_out + 3 * n_sym;
    const double scale = scale_mul * (kind == SKB_STOKESLET ? 1.0 : -3.0) / (8.0 * M_PI);
    cudaStream_t st_std = st;
    if (n_sym > 0 && !aux_stream)
        CUDA_TRY(cudaStreamCreateWithFlags(aux_stream.out(), cudaStreamNonBlocking));
    if (n_sym > 0 && n_trg_std > 0) { // fork: the remainder fills the SMs the symmetric kernel's tail leaves idle
        CUDA_TRY(cudaEventRecord(ev_fork, st));
        CUDA_TRY(cudaStreamWaitEvent(aux_stream, ev_fork, 0));
        st_std = aux_stream;
    }
    LaunchPlan plan{};
    // the long symmetric kernel is launched first so that the remainder's CTAs are dispatched into its tail
    if (n_sym > 0)
        SKB_TRY(sym_eval(*this, opts.d_u_sym ? opts.d_u_sym : d_u_out,
                         opts.sym_accumulate >= 0 ? opts.sym_accumulate : accumulate, st, scale_mul, launches));
    if (n_trg_std > 0) {
        const int *d_src_ids = nullptr, *d_trg_ids = nullptr;
        if (excl && n_sym == 0) { // the whole target list goes through the plain kernel: it needs per-target ids
            if (s.excl_trg_n != n_trg) {
                SKB_TRY(s.excl_trg.ensure((size_t)n_trg * sizeof(int)));
                excl_target_ids_kernel<<<(unsigned)((n_trg + bs - 1) / bs), bs, 0, st_std>>>(
                    (const int *)s.excl_ids.ptr, s.n, trg_begin, n_trg, (int *)s.excl_trg.ptr);
                CUDA_TRY(cudaGetLastError());
                count_launch(1);
                s.excl_trg_n = n_trg;
            }
            d_src_ids = (const int *)s.excl_ids.ptr;
            d_trg_ids = (const int *)s.excl_trg.ptr;
        } // (with the symmetric path the remainder targets are not sources: nothing to exclude there)
        plan = plan_launch(info, kind, n_trg_std, (int)((s.n + kSrcTile - 1) / kSrcTile), force_T, force_S);
        SKB_TRY(partial.ensure((size_t)plan.n_splits * (size_t)n_trg_std * 24));
        SKB_TRY(launch_pair_sum(info, kind, (const double *)s.r.ptr, s.f_cur, s.n, s.n_pad, d_r_trg_std, n_trg_std,
                                (double *)partial.ptr, plan, st_std, d_src_ids, d_trg_ids));
        // 3. combine splits, scale: 1/(8 pi) (kernels.cu:59) or -3/(8 pi) (kernels.cu:26,51)
        SKB_TRY(launch_reduce((const double *)partial.ptr, d_u_std, n_trg_std, plan.n_splits, scale, accumulate,
                              st_std));
        if (launches)
            *launches += 2;
    }
    if (kind == SKB_STOKESLET)
        last_was_sym = n_sym > 0;
    if (n_sym > 0) {
        if (n_trg_std > 0) { // join
            CUDA_TRY(cudaEventRecord(ev_join, aux_stream));
            CUDA_TRY(cudaStreamWaitEvent(st, ev_join, 0));
        }
        plan = sym_launch_plan(s);
    }
    if (ev_k1)
        CUDA_TRY(cudaEventRecord(ev_k1, st));
    if (plan_out)
        *plan_out = plan;
    return SKB_OK;
}

int Evaluator::gradient(int kind, StrengthMode mode, const double *d_f_raw, double two_eta, double *d_g,
                        cudaStream_t st, int *launches, double scale_mul) {
    SourceSet &s = src[kind];
    if (n_trg == 0 || s.n <= 0)
        return SKB_OK;
    SKB_TRY(pack(kind, mode, d_f_raw, two_eta, st, launches));
    const int gkind = kind == SKB_STOKESLET ? kStokesletGrad : kStressletGrad;
    constexpr int kOut = KindTraits<kStokesletGrad>::odim;
    const LaunchPlan plan = plan_launch(info, gkind, n_trg, (int)((s.n + kSrcTile - 1) / kSrcTile), kGradT, 0);
    SKB_TRY(partial.ensure((size_t)plan.n_splits * (size_t)n_trg * kOut * 8));
    SKB_TRY(launch_pair_sum(info, gkind, (const double *)s.r.ptr, s.f_cur, s.n, s.n_pad, (const double *)r_trg.ptr,
                            n_trg, (double *)partial.ptr, plan, st));
    const double scale = scale_mul * (kind == SKB_STOKESLET ? 1.0 : -3.0) / (8.0 * M_PI);
    SKB_TRY(launch_reduce((const double *)partial.ptr, d_g, n_trg, plan.n_splits, scale, 1, st, kOut));
    if (launches)
        *launches += 2;
    return SKB_OK;
}
} // namespace skb

// skb_ctx.cu -- the evaluator contexts of include/skelly_b200.h: one Evaluator per device, with the context's own
// stream, timing events and output buffers, the host copies of the positions that decide a multi-device layout, and the
// NCCL all-gather and reduce-scatter between the devices.  Their C ABI, the stateless reference-shaped entry points and
// the reference-named C++ entry points kernels::stokeslet_direct_gpu_impl / kernels::stresslet_direct_gpu_impl
// (SkellySim include/kernels.hpp:17-20), so the library links in place of src/core/kernels.cu.
//
// No CPU fallback exists here: every path ends in a CUDA launch or an error code.
#include "skb_internal.hpp"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <vector>

using namespace skb;

struct skb_ctx {
    // one device: its evaluator, and the context's own stream, timing events and output buffers
    struct Device {
        Evaluator ev;
        Stream stream;
        Event ev_t0, ev_t1, ev_k0, ev_k1;
        // symmetric multi-device layout: [all n_self leading targets | remainder rows rem_begin.. +rem_count]
        long long rem_begin = 0, rem_count = 0;
        DevBuf u;    // the evaluation's output on this device
        DevBuf u_rs; // reduce-scatter output (this device's chunk of the leading rows)
    };
    ~skb_ctx(); // releases each device's state with that device current
    std::vector<Device> devs;
    long long n_trg = -1;
    // single-process multi-device symmetric layout (host-pointer API): host copies of the positions decide it
    std::vector<double> h_trg, h_src[2];
    bool sym_layout = false;    // devices currently hold the targets in the symmetric layout
    bool layout_dirty = false;  // positions changed since the devices' target layout was decided
    long long n_self = 0;       // leading targets that are the Stokeslet sources
    skb_eval_stats stats{};
    bool kernel_events_pending = false; // device-pointer path: kernel_ms is read back lazily
    void *nccl = nullptr; // NcclGroup*, multi-device contexts only
};

skb_ctx::~skb_ctx() {
    while (!devs.empty()) { // each device's buffers are freed with that device current
        if (devs.back().stream) // (an entry a failed create never reached owns nothing)
            cudaSetDevice(devs.back().ev.info.dev);
        devs.pop_back();
    }
    if (nccl)
        nccl_group_destroy(nccl);
}

// every device's stream has drained
static int sync_devices(skb_ctx *ctx) {
    for (auto &d : ctx->devs) {
        CUDA_TRY(cudaSetDevice(d.ev.info.dev));
        CUDA_TRY(cudaStreamSynchronize(d.stream));
    }
    return SKB_OK;
}

// the host copies of the positions: the targets start with the n Stokeslet sources
static bool targets_lead_with_sources(const skb_ctx *ctx, long long n) {
    return ctx->n_trg >= n && (long long)ctx->h_src[SKB_STOKESLET].size() == 3 * n &&
           std::memcmp(ctx->h_trg.data(), ctx->h_src[SKB_STOKESLET].data(), (size_t)n * 24) == 0;
}

static void set_stats(skb_ctx *ctx, long long n_src, int launches, const LaunchPlan &plan, double k_ms, double t_ms) {
    ctx->stats.kernel_ms = k_ms;
    ctx->stats.total_ms = t_ms;
    ctx->stats.n_pairs = n_src * ctx->n_trg;
    ctx->stats.launches = launches;
    ctx->stats.targets_per_thread = plan.T;
    ctx->stats.source_splits = plan.n_splits;
    ctx->stats.grid_ctas = (int)(plan.grid_x * plan.n_splits);
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
    ctx->devs.resize(n);
    for (int g = 0; g < n; ++g) {
        skb_ctx::Device &d = ctx->devs[g];
        const int dev = ids ? ids[g] : g;
        if (dev < 0 || dev >= n_dev)
            return set_error(SKB_ERR_INVALID, "device id %d out of range", dev);
        SKB_TRY(prepare_device(dev));
        CUDA_TRY(cudaStreamCreateWithFlags(d.stream.out(), cudaStreamNonBlocking));
        SKB_TRY(d.ev.init(query_device(dev)));
        d.ev.layout = n > 1 ? Evaluator::kBlocks : Evaluator::kOwn;
        CUDA_TRY(cudaEventCreate(d.ev_t0.out()));
        CUDA_TRY(cudaEventCreate(d.ev_t1.out()));
        CUDA_TRY(cudaEventCreate(d.ev_k0.out()));
        CUDA_TRY(cudaEventCreate(d.ev_k1.out()));
    }
    if (n > 1)
        SKB_TRY(nccl_group_create(ctx->devs.size(), [&](int g) { return ctx->devs[g].ev.info.dev; }, &ctx->nccl));
    *out = ctx.release();
    return SKB_OK;
}

extern "C" {

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
    for (auto &d : ctx->devs) {
        d.ev.force_T = T;
        d.ev.force_S = S;
    }
    return SKB_OK;
}

int skb_ctx_set_symmetric(skb_ctx *ctx, int mode) {
    if (!ctx || mode < -1 || mode > 1)
        return set_error(SKB_ERR_INVALID, "skb_ctx_set_symmetric: mode must be -1 (auto), 0 (off) or 1 (on)");
    for (auto &d : ctx->devs)
        d.ev.sym_mode = mode;
    return SKB_OK;
}

int skb_ctx_last_eval_was_symmetric(const skb_ctx *ctx, int *yes) {
    if (!ctx || !yes)
        return set_error(SKB_ERR_INVALID, "skb_ctx_last_eval_was_symmetric: NULL");
    *yes = ctx->devs[0].ev.last_was_sym ? 1 : 0; // (every device of a layout decides alike)
    return SKB_OK;
}

int skb_ctx_set_sym_partition(skb_ctx *ctx, int part, int n_parts) {
    if (!ctx || n_parts < 1 || part < 0 || part >= n_parts)
        return set_error(SKB_ERR_INVALID, "skb_ctx_set_sym_partition: need 0 <= part < n_parts");
    if (ctx->devs.size() != 1)
        return set_error(SKB_ERR_INVALID, "skb_ctx_set_sym_partition: single-GPU contexts only");
    ctx->devs[0].ev.sym_part = part;
    ctx->devs[0].ev.sym_parts = n_parts;
    return SKB_OK;
}

int skb_ctx_last_sym_kernel(const skb_ctx *ctx, double *ms, int64_t *pairs) {
    if (!ctx)
        return set_error(SKB_ERR_INVALID, "skb_ctx_last_sym_kernel: NULL");
    return ctx->devs[0].ev.last_sym_kernel(ms, pairs);
}

int skb_last_eval_stats(const skb_ctx *ctx, skb_eval_stats *out) {
    if (!ctx || !out)
        return set_error(SKB_ERR_INVALID, "skb_last_eval_stats: NULL");
    *out = ctx->stats;
    if (ctx->kernel_events_pending) {
        // asynchronous evaluation: the events are valid once the caller's stream has passed them
        const skb_ctx::Device &d = ctx->devs[0];
        float ms = 0;
        cudaSetDevice(d.ev.info.dev);
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
        Evaluator &e = ctx->devs[g].ev;
        e.trg_begin = std::min(n_trg, g * chunk);
        e.n_trg = std::min(n_trg, (g + 1) * chunk) - e.trg_begin;
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
    skb_ctx::Device &d = ctx->devs[0];
    ctx->n_trg = n_trg;
    SKB_TRY(d.ev.set_targets(r_trg, n_trg, on_device, on_device ? user : d.stream));
    if (n_trg > 0)
        SKB_TRY(d.u.ensure((size_t)n_trg * 24));
    return on_device ? SKB_OK : sync_devices(ctx);
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
    const Evaluator &e0 = ctx->devs[0].ev;
    const long long n_sl = e0.src[SKB_STOKESLET].n, n_dl = e0.src[SKB_STRESSLET].n;
    const long long block = sym_block_nodes();
    bool want = e0.sym_mode != 0 && n_dl <= 0 && n_sl >= (e0.sym_mode == 1 ? 2 * block : 4096) &&
                targets_lead_with_sources(ctx, n_sl);
    if (want) {
        const long long n_pad = e0.src[SKB_STOKESLET].n_pad;
        if (((n_pad / block + P - 1) / P) * n_pad * 24 > sym_mem_budget())
            want = false;
    }
    ctx->sym_layout = want;
    ctx->n_self = want ? n_sl : 0;
    if (!want) {
        partition_targets(ctx, n_trg);
        for (auto &d : ctx->devs) {
            d.ev.sym_part = 0;
            d.ev.sym_parts = 1;
            d.rem_begin = d.rem_count = 0;
        }
    } else {
        const long long n_rem = n_trg - n_sl, chunk = (n_rem + P - 1) / P;
        for (long long g = 0; g < P; ++g) {
            skb_ctx::Device &d = ctx->devs[g];
            d.rem_begin = std::min(n_rem, g * chunk);
            d.rem_count = std::min(n_rem, (g + 1) * chunk) - d.rem_begin;
            d.ev.trg_begin = 0;
            d.ev.n_trg = n_sl + d.rem_count;
            d.ev.sym_part = (int)g;
            d.ev.sym_parts = (int)P;
        }
    }
    for (auto &d : ctx->devs) {
        Evaluator &e = d.ev;
        e.layout = want ? Evaluator::kShared : Evaluator::kBlocks;
        e.src[0].sym.self_state = want ? 1 : 0; // decided on the host copies
        if (e.n_trg == 0)
            continue;
        CUDA_TRY(cudaSetDevice(e.info.dev));
        const long long chunk_f = want ? (ctx->n_self + P - 1) / P : 0;
        const long long u_rows = std::max(e.n_trg, chunk_f * P);
        SKB_TRY(e.r_trg.ensure((size_t)e.n_trg * 24));
        SKB_TRY(d.u.ensure((size_t)u_rows * 24));
        if (want) {
            SKB_TRY(d.u_rs.ensure((size_t)chunk_f * 24));
            CUDA_TRY(cudaMemcpyAsync(e.r_trg.ptr, ctx->h_trg.data(), (size_t)ctx->n_self * 24, cudaMemcpyHostToDevice,
                                     d.stream));
            if (d.rem_count > 0)
                CUDA_TRY(cudaMemcpyAsync((double *)e.r_trg.ptr + 3 * ctx->n_self,
                                         ctx->h_trg.data() + 3 * (ctx->n_self + d.rem_begin), (size_t)d.rem_count * 24,
                                         cudaMemcpyHostToDevice, d.stream));
        } else {
            CUDA_TRY(cudaMemcpyAsync(e.r_trg.ptr, ctx->h_trg.data() + 3 * e.trg_begin, (size_t)e.n_trg * 24,
                                     cudaMemcpyHostToDevice, d.stream));
        }
    }
    SKB_TRY(sync_devices(ctx));
    ctx->layout_dirty = false;
    return SKB_OK;
}

static int set_sources_impl(skb_ctx *ctx, int kind, const double *r_src, long long n_src, bool on_device,
                            cudaStream_t user) {
    if (!ctx)
        return set_error(SKB_ERR_INVALID, "set_sources: NULL ctx");
    SKB_TRY(check_sources(kind, r_src, n_src));
    if (on_device && ctx->devs.size() != 1)
        return set_error(SKB_ERR_INVALID, "device-pointer entry points need a single-GPU context");
    const long long P = (long long)ctx->devs.size();
    if (!on_device && P > 1) {
        ctx->h_src[kind].assign(r_src, r_src + 3 * n_src);
        ctx->layout_dirty = true;
    }
    for (auto &d : ctx->devs)
        SKB_TRY(d.ev.set_sources(kind, r_src, n_src, on_device, on_device ? user : d.stream, P));
    return on_device ? SKB_OK : sync_devices(ctx);
}

// ------------------------------------------------------------------------------------------------
// evaluation
// ------------------------------------------------------------------------------------------------
// host-pointer evaluation over all devices of the context
static int eval_host(skb_ctx *ctx, int kind, StrengthMode mode, const double *f_src, double eta, double *u_trg,
                     int accumulate) {
    if (!ctx)
        return set_error(SKB_ERR_INVALID, "eval: NULL ctx");
    SKB_TRY(check_kind(kind));
    if (ctx->n_trg < 0)
        return set_error(SKB_ERR_STATE, "eval: skb_set_targets has not been called");
    const long long n_src = ctx->devs[0].ev.src[kind].n;
    if (n_src < 0)
        return set_error(SKB_ERR_STATE, "eval: skb_set_sources(kind=%d) has not been called", kind);
    if ((n_src > 0 && !f_src) || (ctx->n_trg > 0 && !u_trg))
        return set_error(SKB_ERR_INVALID, "eval: NULL strength or output pointer");
    if (mode == kNormalDensity && n_src > 0 && !ctx->devs[0].ev.src[kind].has_normals)
        return set_error(SKB_ERR_STATE, "eval_double_layer: skb_set_source_normals has not been called");
    SKB_TRY(update_layout(ctx));
    if (kind == SKB_STOKESLET && ctx->devs.size() > 1 && ctx->devs[0].ev.src[kind].excl &&
        !targets_lead_with_sources(ctx, n_src))
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
        skb_ctx::Device &d = ctx->devs[g];
        CUDA_TRY(cudaSetDevice(d.ev.info.dev));
        CUDA_TRY(cudaEventRecord(d.ev_t0, d.stream));
        SourceSet &s = d.ev.src[kind];
        const long long b = std::min(n_src, g * chunk), e = std::min(n_src, (g + 1) * chunk);
        if (e > b)
            CUDA_TRY(cudaMemcpyAsync((double *)s.f_raw.ptr + (size_t)g * chunk * fdim, f_src + (size_t)b * fdim,
                                     (size_t)(e - b) * fdim * 8, cudaMemcpyHostToDevice, d.stream));
    }
    if (P > 1) {
        std::vector<void *> bufs(P);
        std::vector<cudaStream_t> sts(P);
        for (long long g = 0; g < P; ++g) {
            bufs[g] = ctx->devs[g].ev.src[kind].f_raw.ptr;
            sts[g] = ctx->devs[g].stream;
        }
        SKB_TRY(nccl_group_allgather_inplace(ctx->nccl, bufs.data(), (size_t)chunk * fdim, sts.data()));
    }
    // stage 2: every device evaluates its targets against all sources
    const long long chunk_f = sym_layout ? (n_self + P - 1) / P : 0; // reduce-scatter slot (leading rows per device)
    for (long long g = 0; g < P; ++g) {
        skb_ctx::Device &d = ctx->devs[g];
        Evaluator &ev = d.ev;
        if (ev.n_trg == 0)
            continue;
        CUDA_TRY(cudaSetDevice(ev.info.dev));
        if (!sym_layout) {
            if (accumulate)
                CUDA_TRY(cudaMemcpyAsync(d.u.ptr, u_trg + 3 * ev.trg_begin, (size_t)ev.n_trg * 24,
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
        SKB_TRY(ev.eval(kind, mode, (const double *)ev.src[kind].f_raw.ptr, 2.0 * eta, (double *)d.u.ptr, accumulate,
                        d.stream, &launches, g == 0 ? &plan : nullptr, 1.0, EvalOpts(), d.ev_k0, d.ev_k1));
        if (!sym_layout) {
            CUDA_TRY(cudaMemcpyAsync(u_trg + 3 * ev.trg_begin, d.u.ptr, (size_t)ev.n_trg * 24, cudaMemcpyDeviceToHost,
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
            skb_ctx::Device &d = ctx->devs[g];
            CUDA_TRY(cudaSetDevice(d.ev.info.dev));
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
        skb_ctx::Device &d = ctx->devs[g];
        CUDA_TRY(cudaSetDevice(d.ev.info.dev));
        CUDA_TRY(cudaStreamSynchronize(d.stream));
        if (d.ev.n_trg == 0)
            continue;
        float ms = 0;
        if (n_src > 0 && cudaEventElapsedTime(&ms, d.ev_k0, d.ev_k1) == cudaSuccess)
            k_ms = std::max(k_ms, (double)ms);
        if (cudaEventElapsedTime(&ms, d.ev_t0, d.ev_t1) == cudaSuccess)
            t_ms = std::max(t_ms, (double)ms);
    }
    ctx->kernel_events_pending = false;
    set_stats(ctx, n_src, launches, plan, k_ms, t_ms);
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
    for (auto &d : ctx->devs)
        SKB_TRY(d.ev.set_normals(normals, n_src, d.stream));
    return sync_devices(ctx);
}

int skb_set_source_exclusion_ids(skb_ctx *ctx, const int32_t *ids, int64_t n_src) {
    if (!ctx)
        return set_error(SKB_ERR_INVALID, "skb_set_source_exclusion_ids: NULL ctx");
    for (auto &d : ctx->devs)
        SKB_TRY(d.ev.set_exclusion_ids(ids, n_src, d.stream));
    return sync_devices(ctx);
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
    skb_ctx::Device &d = ctx->devs[0];
    Evaluator &ev = d.ev;
    if (ctx->n_trg < 0 || ev.src[kind].n < 0)
        return set_error(SKB_ERR_STATE, "eval_device: targets / sources not set");
    if ((ev.src[kind].n > 0 && !d_f_src) || (ctx->n_trg > 0 && !d_u_trg))
        return set_error(SKB_ERR_INVALID, "eval_device: NULL pointer");
    CUDA_TRY(cudaSetDevice(ev.info.dev));
    cudaStream_t st = (cudaStream_t)stream; // verbatim: 0 is CUDA's legacy default stream
    int launches = 0;
    LaunchPlan plan{};
    SKB_TRY(ev.eval(kind, kRaw, d_f_src, 0.0, d_u_trg, accumulate, st, &launches, &plan, 1.0, EvalOpts(), d.ev_k0,
                    d.ev_k1));
    ctx->kernel_events_pending = ev.src[kind].n > 0 && ev.n_trg > 0;
    set_stats(ctx, ev.src[kind].n, launches, plan, 0, 0);
    return SKB_OK;
}

int skb_sync(skb_ctx *ctx) {
    if (!ctx)
        return set_error(SKB_ERR_INVALID, "skb_sync: NULL ctx");
    return sync_devices(ctx);
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
    skb_ctx::Device &d = ctx->devs[0];
    CUDA_TRY(cudaSetDevice(d.ev.info.dev));
    const int blocks = d.ev.info.num_sms * 8, threads = 256, iters = 1 << 15;
    SKB_TRY(d.ev.scratch.ensure((size_t)blocks * threads * 8));
    double best = 0;
    for (int rep = 0; rep < 5; ++rep) {
        CUDA_TRY(cudaEventRecord(d.ev_k0, d.stream));
        SKB_TRY(launch_fp64_probe((double *)d.ev.scratch.ptr, blocks, threads, iters, d.stream));
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

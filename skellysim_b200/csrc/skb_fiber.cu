// skb_fiber.cu -- the per-fiber dense operators of a flow (FiberOps, skb_internal.hpp): the class matrices and their one
// device table, the plan of the own fibers, the caller's operators and inverse or their device build (fiber_build.cuh),
// the launches of fiber_gemv_kernel (fiber_ops.cuh), and the fiber block of the RHS (fiber_rhs.cuh) with per-fiber
// tables of its own.  Knows nothing of skb_flow: the fiber operators' entry points in skb_system.cu hand it the own
// fibers.
#include "fiber_build.cuh"
#include "fiber_ops.cuh"
#include "fiber_rhs.cuh"
#include "step_kernels.cuh"
#include "skb_internal.hpp"
#include "../../include/skelly_b200_flow.h"

#include <algorithm>
#include <cmath>

using namespace skb;

// fiber_gemv_kernel's dynamic shared memory: the plan refuses more, prepare_fiber_kernels allows this much
static constexpr size_t kGemvSmemMax = kFiberGemvSmemMax;

// Where the operators of the own fibers live (GEMV items, offsets into A_, force_operator_ and the class table) and a
// build's tables: per fiber, per assembly CTA (a tile of columns), per inverse launch (node count)
struct FiberOps::Plan {
    std::vector<long long> cD, cP, cR;        // per own fiber: its class's D_1_0, P, ranges
    std::vector<FiberGemvItem> itA, itF;
    long long offA = 0, offF = 0;
    std::vector<FiberItem> items;
    std::vector<FiberTileItem> tiles;
    std::vector<double> lp;
    std::vector<int> plus;
    std::map<int, std::vector<long long>> inv_by_n;
    std::vector<long long> inv_off;
    size_t smem = 0;
};

// per line k < lines: first / one-past-last t < len with m[k * ks + t * ts] != 0, (0, 0) for a zero line
static void nonzero_ranges(const double *m, int lines, size_t ks, int len, size_t ts, std::vector<int2> &out) {
    for (int k = 0; k < lines; ++k) {
        int t0 = len, t1 = 0;
        for (int t = 0; t < len; ++t)
            if (m[k * ks + t * ts] != 0.0) {
                t0 = std::min(t0, t);
                t1 = t + 1;
            }
        out.push_back(t1 > t0 ? make_int2(t0, t1) : make_int2(0, 0));
    }
}

int FiberOps::set_class(int n_nodes, const double *D_1_0, const double *P_downsample_bc, cudaStream_t st) {
    if (n_nodes < 4) // bc_start_i = 4n - 14 must leave room for the 14 boundary rows (ffd.cpp:279)
        return set_error(SKB_ERR_INVALID, "skb_flow_set_fiber_class: n_nodes = %d (need >= 4)", n_nodes);
    const size_t n = (size_t)n_nodes;
    FiberClass &c = classes[n_nodes];
    c.D.assign(D_1_0, D_1_0 + n * n);
    c.P.assign(P_downsample_bc, P_downsample_bc + (4 * n - 14) * 4 * n);
    ready_ = false; // the offsets of the other classes may have moved
    return upload_classes(st);
}

int FiberOps::set_class_derivatives(int n_nodes, const double *D_2_0, const double *D_3_0, const double *D_4_0,
                                    cudaStream_t st) {
    if (n_nodes < kBuildMinNodes || n_nodes > kBuildMaxNodes)
        return set_error(SKB_ERR_INVALID, "skb_flow_set_fiber_class_derivatives: n_nodes = %d (the device build takes "
                                          "%d <= n <= %d)", n_nodes, kBuildMinNodes, kBuildMaxNodes);
    const size_t nn = (size_t)n_nodes * n_nodes;
    FiberClass &c = classes[n_nodes];
    c.D234.assign(D_2_0, D_2_0 + nn);
    c.D234.insert(c.D234.end(), D_3_0, D_3_0 + nn);
    c.D234.insert(c.D234.end(), D_4_0, D_4_0 + nn);
    return c.D.empty() ? SKB_OK : upload_classes(st); // without set_class(n) yet: its block is written then
}

// classes -> class_mats / class_ranges / class_off, in order of n.  Per class also the non-zero column range of every
// row of P_downsample_bc (block diagonal in the reference, ffd.cpp:551-555: the kernels walk the range only) and the
// non-zero row range of every column of D_1_0.
int FiberOps::upload_classes(cudaStream_t st) {
    std::vector<double> mats;
    std::vector<int2> ranges;
    class_off.clear();
    for (const auto &kv : classes) {
        if (kv.second.D.empty()) // only set_class_derivatives was called for this n
            continue;
        const int nn = kv.first, bc = 4 * nn - 14;
        class_off[nn] = {(long long)mats.size(), (long long)ranges.size()};
        mats.insert(mats.end(), kv.second.D.begin(), kv.second.D.end());
        mats.insert(mats.end(), kv.second.P.begin(), kv.second.P.end());
        if (kv.second.D234.empty())
            mats.resize(mats.size() + 3 * (size_t)nn * nn, 0.0);
        else
            mats.insert(mats.end(), kv.second.D234.begin(), kv.second.D234.end());
        nonzero_ranges(kv.second.P.data(), bc, 1, 4 * nn, bc, ranges);
        // D_1_0 (n x n, column-major): non-zero row range of every column (banded)
        nonzero_ranges(kv.second.D.data(), nn, nn, nn, 1, ranges);
    }
    CUDA_TRY(cudaDeviceSynchronize()); // the GEMVs, the build and the RHS may still read the table, on any stream
    SKB_TRY(class_mats.upload(mats.data(), mats.size() * 8, st));
    SKB_TRY(class_ranges.upload(ranges.data(), ranges.size() * sizeof(int2), st));
    CUDA_TRY(cudaStreamSynchronize(st)); // complete before any later launch, on any stream
    return SKB_OK;
}

// derivatives: the device build's and the RHS's needs (class derivatives, n within the build's range)
bool FiberOps::buildable(int n) const {
    const auto it = classes.find(n);
    return n >= kBuildMinNodes && n <= kBuildMaxNodes && it != classes.end() && !it->second.D.empty() &&
           !it->second.D234.empty();
}
int FiberOps::build_min_nodes() { return kBuildMinNodes; }
int FiberOps::build_max_nodes() { return kBuildMaxNodes; }

int FiberOps::check_class(int f, int n, bool derivatives) const {
    auto it = classes.find(n);
    if (it == classes.end() || it->second.D.empty())
        return set_error(SKB_ERR_INVALID, "fiber %d has %d nodes but skb_flow_set_fiber_class(%d, ...) was never "
                                          "called", f, n, n);
    if (derivatives && (n < kBuildMinNodes || n > kBuildMaxNodes))
        return set_error(SKB_ERR_INVALID, "fiber %d has %d nodes: the device build takes %d <= n <= %d", f, n,
                         kBuildMinNodes, kBuildMaxNodes);
    if (derivatives && it->second.D234.empty())
        return set_error(SKB_ERR_INVALID, "fiber %d has %d nodes but skb_flow_set_fiber_class_derivatives(%d, ...) "
                                          "was never called", f, n, n);
    return SKB_OK;
}

int FiberOps::derivative_offset(int f, int n, long long *off) const {
    SKB_TRY(check_class(f, n, true));
    *off = class_off.at(n).first + (long long)n * n + (4LL * n - 14) * 4 * n; // past D_1_0 and P_downsample_bc
    return SKB_OK;
}

// a_off / f_off are the build's
int FiberOps::item(const OwnFibers &own, int f, bool derivatives, FiberItem &it) const {
    const int n = own.n[f];
    SKB_TRY(check_class(f, n, derivatives));
    const auto &co = class_off.at(n);
    it = FiberItem{0, 0, own.off[f], own.off[f] - own.off[own.f0], co.first, co.second, n, f};
    return SKB_OK;
}

// length_prev: checked per fiber when given; build: the parameters of a device build (class derivatives needed, n
// within the build's range), whose tables are planned too
int FiberOps::plan(const OwnFibers &own, const double *length_prev, const skb_fiber_params *build, Plan &pl) {
    const int f0 = own.f0, nfib = own.count();
    pl.cD.resize((size_t)nfib), pl.cP.resize((size_t)nfib), pl.cR.resize((size_t)nfib);
    int max_n = 0;
    for (int f = 0; f < nfib; ++f) {
        FiberItem it;
        SKB_TRY(item(own, f0 + f, build != nullptr, it));
        if (length_prev && !(length_prev[f] > 0))
            return set_error(SKB_ERR_INVALID, "fiber %d: length_prev = %g", f0 + f, length_prev[f]);
        const int n = it.n;
        const long long node_off = it.own_node; // x / fw / v / res of the own fibers are indexed from their first node
        pl.cD[f] = it.cls;
        pl.cP[f] = it.cls + (long long)n * n;
        pl.cR[f] = it.rng;
        max_n = std::max(max_n, n);
        if (build) {
            it.a_off = pl.offA;
            it.f_off = pl.offF;
            pl.items.push_back(it);
            for (int c = 0; c < 4 * n; c += build_tile_cols(n))
                pl.tiles.push_back(FiberTileItem{f, c});
            pl.smem = std::max(pl.smem, build_smem_bytes(n));
            pl.inv_by_n[n].push_back(pl.offA);
            pl.lp.push_back(build[f].length_prev);
            pl.plus.push_back(build[f].plus_hinged);
        }
        for (int r0 = 0; r0 < 4 * n; r0 += kFiberGemvRows)
            pl.itA.push_back(FiberGemvItem{pl.offA, 4 * node_off, 4 * node_off, 4 * n, 4 * n, r0, n, f, 0});
        for (int r0 = 0; r0 < 3 * n; r0 += kFiberGemvRows)
            pl.itF.push_back(FiberGemvItem{pl.offF, 4 * node_off, node_off, 3 * n, 4 * n, r0, n, f, 0});
        pl.offA += 16LL * n * n;
        pl.offF += 12LL * n * n;
    }
    for (const auto &kv : pl.inv_by_n)
        pl.inv_off.insert(pl.inv_off.end(), kv.second.begin(), kv.second.end());
    // x (4n) + slice partials + vT (4n) + s (n)
    gemv_smem = ((size_t)2 * ((4 * max_n + 1) & ~1) + kFiberGemvThreads + (size_t)max_n) * sizeof(double);
    if (gemv_smem > kGemvSmemMax)
        return set_error(SKB_ERR_INVALID, "fiber with %d nodes exceeds the shared-memory fiber operator kernels", max_n);
    return SKB_OK;
}

// the plan's buffers on the device and room for the operators (on own.stream; the caller synchronises before `pl`
// goes out of scope)
int FiberOps::upload_plan(const OwnFibers &own, const Plan &pl) {
    const cudaStream_t st = own.stream;
    SKB_TRY(op_A.ensure((size_t)pl.offA * 8));
    SKB_TRY(op_F.ensure((size_t)pl.offF * 8));
    SKB_TRY(op_xs.ensure((size_t)own.nodes() * 24));
    SKB_TRY(op_classD.upload(pl.cD.data(), pl.cD.size() * 8, st));
    SKB_TRY(op_classP.upload(pl.cP.data(), pl.cP.size() * 8, st));
    SKB_TRY(op_classR.upload(pl.cR.data(), pl.cR.size() * 8, st));
    SKB_TRY(items_A.upload(pl.itA.data(), pl.itA.size() * sizeof(FiberGemvItem), st));
    SKB_TRY(items_F.upload(pl.itF.data(), pl.itF.size() * sizeof(FiberGemvItem), st));
    return SKB_OK;
}

void FiberOps::commit(const OwnFibers &own, const Plan &pl) {
    f0 = own.f0;
    f1 = own.f1;
    n_nodes = own.nodes();
    n_items_A = (int)pl.itA.size();
    n_items_F = (int)pl.itF.size();
    op_A_elems = pl.offA;
    op_F_elems = pl.offF;
    ops_gen++;
    ready_ = true;
}

int FiberOps::upload(const OwnFibers &own, const double *A, const double *force_operator, const double *xs,
                     const double *length_prev, const int *plus_bc_velocity) {
    ready_ = false;
    const int nfib = own.count();
    if (nfib == 0) { // resident for no fiber; the generation stays
        f0 = own.f0;
        f1 = own.f1;
        n_items_A = n_items_F = 0;
        ready_ = true;
        return SKB_OK;
    }
    Plan pl;
    SKB_TRY(plan(own, length_prev, nullptr, pl));
    SKB_TRY(upload_plan(own, pl));
    SKB_TRY(upload_pageable(op_A.ptr, A, (size_t)pl.offA * 8, own.stream));
    SKB_TRY(upload_pageable(op_F.ptr, force_operator, (size_t)pl.offF * 8, own.stream));
    CUDA_TRY(cudaMemcpyAsync(op_xs.ptr, xs, (size_t)own.nodes() * 24, cudaMemcpyHostToDevice, own.stream));
    SKB_TRY(op_len.upload(length_prev, (size_t)nfib * 8, own.stream));
    SKB_TRY(op_plus.upload(plus_bc_velocity, (size_t)nfib * sizeof(int), own.stream));
    CUDA_TRY(cudaStreamSynchronize(own.stream)); // the host vectors above go out of scope
    commit(own, pl);
    return SKB_OK;
}

int FiberOps::upload_inverse(const double *A_inv, cudaStream_t st) {
    if (!ready_)
        return set_error(SKB_ERR_INVALID, "skb_flow_set_fiber_preconditioner: call skb_flow_set_fiber_operators "
                                          "first (it defines the fibers and their order)");
    if (op_A_elems > 0) {
        if (!A_inv)
            return set_error(SKB_ERR_INVALID, "skb_flow_set_fiber_preconditioner: NULL argument");
        SKB_TRY(op_Ainv.ensure((size_t)op_A_elems * 8));
        SKB_TRY(upload_pageable(op_Ainv.ptr, A_inv, (size_t)op_A_elems * 8, st));
    }
    precond_gen = ops_gen;
    return SKB_OK;
}

static int check_params(const OwnFibers &own, const skb_fiber_params *params) {
    static_assert(sizeof(skb_fiber_params) == 48 && sizeof(FiberParamsDev) == 48, "skb_fiber_params layout");
    for (int f = 0; f < own.count(); ++f) {
        const skb_fiber_params &p = params[f];
        if (!(p.length_prev > 0) || !(p.radius > 0))
            return set_error(SKB_ERR_INVALID, "fiber %d: length_prev = %g, radius = %g (both must be > 0)",
                             own.f0 + f, p.length_prev, p.radius);
        if ((p.minus_clamped != 0 && p.minus_clamped != 1) || (p.plus_hinged != 0 && p.plus_hinged != 1))
            return set_error(SKB_ERR_INVALID, "fiber %d: minus_clamped = %d, plus_hinged = %d (each must be 0 or 1)",
                             own.f0 + f, p.minus_clamped, p.plus_hinged);
    }
    return SKB_OK;
}

int FiberOps::build(const OwnFibers &own, const skb_fiber_params *params, double dt, double eta, int *launches,
                    const std::function<int(const Step &stage, const Step &launch)> &frame, bool with_inverse) {
    ready_ = false;
    const int nfib = own.count();
    SKB_TRY(check_params(own, params));
    Plan b;
    if (nfib > 0)
        SKB_TRY(plan(own, nullptr, params, b));
    const cudaStream_t st = own.stream;
    auto stage = [&]() -> int {
        SKB_TRY(upload_plan(own, b));
        if (with_inverse)
            SKB_TRY(op_Ainv.ensure((size_t)b.offA * 8));
        SKB_TRY(op_len.upload(b.lp.data(), b.lp.size() * 8, st));
        SKB_TRY(op_plus.upload(b.plus.data(), b.plus.size() * sizeof(int), st));
        SKB_TRY(bld_params.upload(params, (size_t)nfib * sizeof(skb_fiber_params), st));
        SKB_TRY(bld_items.upload(b.items.data(), b.items.size() * sizeof(FiberItem), st));
        SKB_TRY(bld_tiles.upload(b.tiles.data(), b.tiles.size() * sizeof(FiberTileItem), st));
        return bld_inv.upload(b.inv_off.data(), b.inv_off.size() * sizeof(long long), st);
    };
    auto launch = [&]() -> int {
        const BuildArgs ba{(const FiberItem *)bld_items.ptr, (const FiberTileItem *)bld_tiles.ptr,
                           (const FiberParamsDev *)bld_params.ptr, (const double *)class_mats.ptr,
                           (const int2 *)class_ranges.ptr, own.r_fib, own.length, dt, eta, (double *)op_A.ptr,
                           (double *)op_F.ptr, (double *)op_xs.ptr};
        fiber_assemble_kernel<<<(unsigned)b.tiles.size(), kBuildThreads, b.smem, st>>>(ba);
        SKB_TRY(launched(launches));
        if (!with_inverse)
            return SKB_OK;
        size_t first = 0;
        for (const auto &kv : b.inv_by_n) {
            const int m = 4 * kv.first, cs = inverse_cluster_size(m);
            cudaLaunchConfig_t cfg = {};
            cudaLaunchAttribute attr[1];
            attr[0].id = cudaLaunchAttributeClusterDimension;
            attr[0].val.clusterDim.x = (unsigned)cs;
            attr[0].val.clusterDim.y = attr[0].val.clusterDim.z = 1;
            cfg.gridDim = dim3((unsigned)(kv.second.size() * cs));
            cfg.blockDim = dim3(kInverseThreads);
            cfg.dynamicSmemBytes = inverse_smem_bytes(m, cs);
            cfg.stream = st;
            cfg.attrs = attr;
            cfg.numAttrs = 1;
            void (*kern)(const long long *, const double *, double *, int) =
                m <= 128 ? fiber_inverse_kernel<4> : fiber_inverse_kernel<16>;
            if (cs > 1) {
                int n_clusters = 0, dev = -1;
                CUDA_TRY(cudaOccupancyMaxActiveClusters(&n_clusters, kern, &cfg));
                if (n_clusters < 1) {
                    cudaGetDevice(&dev);
                    return set_error(SKB_ERR_CUDA, "skb_flow_build_fiber_operators: a cluster of %d CTAs x %zu bytes "
                                     "of shared memory (n = %d) does not fit on device %d", cs, cfg.dynamicSmemBytes,
                                     kv.first, dev);
                }
            }
            CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, (const long long *)bld_inv.ptr + first, (const double *)op_A.ptr,
                                        (double *)op_Ainv.ptr, m));
            SKB_TRY(launched(launches));
            first += kv.second.size();
        }
        return SKB_OK;
    };
    if (nfib > 0)
        SKB_TRY(frame(stage, launch)); // (returns once the stream has drained: the plan's tables may go)
    commit(own, b);
    if (with_inverse)
        precond_gen = ops_gen; // the inverse belongs to these operators
    return SKB_OK;
}

// The tables go up from pageable host memory: cudaMemcpyAsync returns once they are staged, so `frame` need not wait
// for the kernel.
int FiberOps::rhs(const OwnFibers &own, const skb_fiber_params *params, const double *v_growth,
                  const double *force_scale, const double *d_v, const double *d_f, double dt, double eta,
                  double *d_rhs, int *launches, const std::function<int(const Step &stage, const Step &launch)> &frame) {
    const int nfib = own.count();
    if (nfib == 0)
        return SKB_OK;
    SKB_TRY(check_params(own, params));
    std::vector<FiberItem> items((size_t)nfib);
    std::vector<double2> growth((size_t)nfib);
    int max_n = 0;
    for (int f = 0; f < nfib; ++f) {
        SKB_TRY(item(own, own.f0 + f, true, items[(size_t)f]));
        const double vg = v_growth ? v_growth[f] : 0.0, fs = force_scale ? force_scale[f] : 0.0;
        if (!std::isfinite(vg) || !std::isfinite(fs))
            return set_error(SKB_ERR_INVALID, "fiber %d: v_growth = %g, force_scale = %g (both must be finite)",
                             own.f0 + f, vg, fs);
        growth[(size_t)f] = make_double2(vg, fs);
        max_n = std::max(max_n, items[(size_t)f].n);
    }
    const cudaStream_t st = own.stream;
    auto stage = [&]() -> int {
        if (rhs_pending) // the previous call's kernel, on whichever stream, still reads these tables
            CUDA_TRY(cudaStreamWaitEvent(st, rhs_done, 0));
        SKB_TRY(rhs_items.upload(items.data(), items.size() * sizeof(FiberItem), st));
        SKB_TRY(rhs_params.upload(params, (size_t)nfib * sizeof(skb_fiber_params), st));
        return rhs_growth.upload(growth.data(), growth.size() * sizeof(double2), st);
    };
    auto launch = [&]() -> int {
        const RhsArgs ra{(const FiberItem *)rhs_items.ptr, (const FiberParamsDev *)rhs_params.ptr,
                         (const double2 *)rhs_growth.ptr, (const double *)class_mats.ptr,
                         (const int2 *)class_ranges.ptr, own.r_fib, own.length, d_v, d_f, force_scale != nullptr, dt, eta, d_rhs};
        fiber_rhs_kernel<<<(unsigned)nfib, kRhsThreads, rhs_smem_bytes(max_n), st>>>(ra);
        SKB_TRY(launched(launches));
        if (!rhs_done)
            CUDA_TRY(cudaEventCreateWithFlags(rhs_done.out(), cudaEventDisableTiming));
        CUDA_TRY(cudaEventRecord(rhs_done, st));
        rhs_pending = true;
        return SKB_OK;
    };
    return frame(stage, launch);
}

int FiberOps::check_step(const OwnFibers &own, const skb_fiber_params *params, const double *v_growth,
                         const double *force_scale) const {
    SKB_TRY(check_params(own, params));
    for (int f = 0; f < own.count(); ++f) {
        SKB_TRY(check_class(own.f0 + f, own.n[own.f0 + f], true));
        const double vg = v_growth ? v_growth[f] : 0.0, fs = force_scale ? force_scale[f] : 0.0;
        if (!std::isfinite(vg) || !std::isfinite(fs))
            return set_error(SKB_ERR_INVALID, "fiber %d: v_growth = %g, force_scale = %g (both must be finite)",
                             own.f0 + f, vg, fs);
    }
    return SKB_OK;
}

int FiberOps::step_items(const OwnFibers &own, std::vector<StepItem> &items) const {
    items.assign((size_t)own.count(), StepItem{});
    for (int f = 0; f < own.count(); ++f) {
        const int g = own.f0 + f, n = own.n[g];
        SKB_TRY(check_class(g, n, false));
        if (n > kStepMaxNodes)
            return set_error(SKB_ERR_INVALID, "fiber %d has %d nodes: the fiber step takes at most %d", g, n,
                             kStepMaxNodes);
        const auto &co = class_off.at(n);
        StepItem &it = items[(size_t)f];
        it.node = own.off[g] - own.off[own.f0];
        it.d1 = co.first;
        it.rng = co.second + 4LL * n - 14; // past P_downsample_bc's row ranges
        it.n = n;
    }
    return SKB_OK;
}

int FiberOps::size_build(const OwnFibers &own) {
    cudaFuncAttributes fa;
    CUDA_TRY(cudaFuncGetAttributes(&fa, fiber_assemble_kernel));
    const int nfib = own.count();
    for (int f = own.f0; f < own.f1; ++f) { // a class the build lacks: nothing to size, the build refuses later
        const auto it = classes.find(own.n[f]);
        if (it == classes.end() || it->second.D.empty() || it->second.D234.empty() || own.n[f] < kBuildMinNodes ||
            own.n[f] > kBuildMaxNodes)
            return SKB_OK;
    }
    const std::array<long long, 4> key = build_key(own);
    if (nfib == 0) {
        build_key_ = key;
        return SKB_OK;
    }
    const std::vector<skb_fiber_params> params((size_t)nfib, skb_fiber_params{});
    Plan b;
    const size_t smem = gemv_smem; // (the plan's GEMV bound belongs to the resident operators until the build)
    const int rc = plan(own, nullptr, params.data(), b);
    gemv_smem = smem;
    SKB_TRY(rc);
    for (auto [buf, bytes] : std::initializer_list<std::pair<DevBuf *, size_t>>{
             {&op_A, (size_t)b.offA * 8}, {&op_F, (size_t)b.offF * 8}, {&op_xs, (size_t)own.nodes() * 24},
             {&op_Ainv, (size_t)b.offA * 8}, {&op_classD, b.cD.size() * 8}, {&op_classP, b.cP.size() * 8},
             {&op_classR, b.cR.size() * 8}, {&items_A, b.itA.size() * sizeof(FiberGemvItem)},
             {&items_F, b.itF.size() * sizeof(FiberGemvItem)}, {&op_len, b.lp.size() * 8},
             {&op_plus, b.plus.size() * sizeof(int)}, {&bld_params, (size_t)nfib * sizeof(skb_fiber_params)},
             {&bld_items, b.items.size() * sizeof(FiberItem)}, {&bld_tiles, b.tiles.size() * sizeof(FiberTileItem)},
             {&bld_inv, b.inv_off.size() * sizeof(long long)}})
        SKB_TRY(buf->ensure(bytes));
    build_key_ = key;
    return SKB_OK;
}

int FiberOps::size_rhs(int n_fibers) {
    const size_t n = (size_t)std::max(n_fibers, 0);
    SKB_TRY(rhs_items.ensure(n * sizeof(FiberItem)));
    SKB_TRY(rhs_params.ensure(n * sizeof(skb_fiber_params)));
    SKB_TRY(rhs_growth.ensure(n * sizeof(double2)));
    if (!rhs_done)
        CUDA_TRY(cudaEventCreateWithFlags(rhs_done.out(), cudaEventDisableTiming));
    return SKB_OK;
}

int FiberOps::ready(const char *who, bool with_inverse) const {
    if (!ready_)
        return set_error(SKB_ERR_INVALID, "%s: call skb_flow_set_fiber_operators after skb_flow_set_fibers / "
                                          "skb_flow_set_fiber_class first", who);
    if (with_inverse && precond_gen != ops_gen)
        return set_error(SKB_ERR_INVALID, "%s: call skb_flow_set_fiber_preconditioner after "
                                          "skb_flow_set_fiber_operators first", who);
    return SKB_OK;
}

// fw = force_operator_ * x per fiber, scattered to 3 x N_f (fcfd.cpp:272-287)
int FiberOps::force(const double *d_x, double *d_fw, cudaStream_t st, int *launches) const {
    if (n_items_F == 0)
        return SKB_OK;
    fiber_gemv_kernel<1><<<n_items_F, kFiberGemvThreads, gemv_smem, st>>>(
        (const FiberGemvItem *)items_F.ptr, (const double *)op_F.ptr, d_x, d_fw, FiberVelArgs{});
    return launched(launches);
}

// res = A_ x - P_downsample_bc vT(v) + xs_vT + y_BC per fiber (ffd.cpp:276-312), one launch; d_vb may be NULL
int FiberOps::matvec(const double *d_x, const double *d_v, const double *d_vb, double *d_res, cudaStream_t st,
                     int *launches) const {
    if (n_items_A == 0)
        return SKB_OK;
    const FiberVelArgs va{(const double *)op_xs.ptr, d_v, (const double *)op_len.ptr, (const int *)op_plus.ptr,
                          (const double *)class_mats.ptr, (const long long *)op_classD.ptr,
                          (const long long *)op_classP.ptr, (const int2 *)class_ranges.ptr,
                          (const long long *)op_classR.ptr, d_vb};
    fiber_gemv_kernel<2><<<n_items_A, kFiberGemvThreads, gemv_smem, st>>>(
        (const FiberGemvItem *)items_A.ptr, (const double *)op_A.ptr, d_x, d_res, va);
    return launched(launches);
}

// y = A_^-1 x per fiber: FiberContainerFiniteDifference::apply_preconditioner (fcfd.cpp:331-339) with the LU solve
// replaced by a GEMV over the explicit inverse (same shapes and item list as A_)
int FiberOps::precondition(const double *d_x, double *d_y, cudaStream_t st, int *launches) const {
    if (n_items_A == 0)
        return SKB_OK;
    fiber_gemv_kernel<0><<<n_items_A, kFiberGemvThreads, gemv_smem, st>>>(
        (const FiberGemvItem *)items_A.ptr, (const double *)op_Ainv.ptr, d_x, d_y, FiberVelArgs{});
    return launched(launches);
}

int skb::launch_gemv(const FiberGemvItem *d_items, int n_items, const double *mats, const double *x, double *y,
                     size_t smem, cudaStream_t st, int *launches) {
    if (n_items == 0)
        return SKB_OK;
    if (smem > kGemvSmemMax)
        return set_error(SKB_ERR_INVALID, "a GEMV of %zu bytes of shared memory exceeds the limit of %zu", smem,
                         kGemvSmemMax);
    fiber_gemv_kernel<0><<<n_items, kFiberGemvThreads, smem, st>>>(d_items, mats, x, y, FiberVelArgs{});
    return launched(launches);
}

int FiberOps::read(double *A, double *force_operator, double *xs, double *A_inv, cudaStream_t st) const {
    if (n_items_A == 0)
        return SKB_OK;
    CUDA_TRY(cudaStreamSynchronize(st));
    if (A)
        CUDA_TRY(cudaMemcpy(A, op_A.ptr, (size_t)op_A_elems * 8, cudaMemcpyDeviceToHost));
    if (force_operator)
        CUDA_TRY(cudaMemcpy(force_operator, op_F.ptr, (size_t)op_F_elems * 8, cudaMemcpyDeviceToHost));
    if (xs)
        CUDA_TRY(cudaMemcpy(xs, op_xs.ptr, (size_t)n_nodes * 24, cudaMemcpyDeviceToHost));
    if (A_inv)
        CUDA_TRY(cudaMemcpy(A_inv, op_Ainv.ptr, (size_t)op_A_elems * 8, cudaMemcpyDeviceToHost));
    return SKB_OK;
}

// (prepare_device, skb_runtime.cu) the GEMVs' dynamic shared memory up to the plan's bound; the inverse's shared
// memory and its non-portable cluster sizes
int skb::prepare_fiber_kernels() {
    for (auto kern : {fiber_gemv_kernel<0>, fiber_gemv_kernel<1>, fiber_gemv_kernel<2>})
        CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kGemvSmemMax));
    for (auto kern : {fiber_inverse_kernel<4>, fiber_inverse_kernel<16>}) {
        CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kInverseSmemMax));
        CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    }
    // loaded now: a group member's system RHS launches it, and a lazy load then could wait behind a peer on the same
    // device spinning on a flag
    cudaFuncAttributes fa;
    CUDA_TRY(cudaFuncGetAttributes(&fa, fiber_rhs_kernel));
    return SKB_OK;
}

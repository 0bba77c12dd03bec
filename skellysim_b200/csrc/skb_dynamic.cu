// skb_dynamic.cu -- System::dynamic_instability (dynamic_instability.cpp:25-194) of a single-device flow
// (include/skelly_b200_flow.h, skb_flow_dynamic_instability): the catastrophe, growth and compaction of the fiber block
// on the device (dynamic_kernels.cuh), the Poisson count and the site picks on the host, and the new fiber set
// installed with everything the next skb_flow_step needs.
#include "dynamic_kernels.cuh"
#include "skb_flow.hpp"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

using namespace skb;

namespace {

constexpr double kPoissonChunk = 256.0; // the largest mean one inversion sums over

// the Poisson count of mean mu by inversion in ceil(mu / 256) equal chunks, chunk i from draw (i, kDiPoisson): within a
// chunk of mean m, p = F = exp(-m), then p *= m / k and F += p until u <= F, k capped at m + 40 sqrt(m) + 40
long long poisson(double mu, uint64_t seed, uint64_t call) {
    if (!(mu > 0))
        return 0;
    const double n_chunks = std::ceil(mu / kPoissonChunk);
    const double m = mu / n_chunks, cap = m + 40.0 * std::sqrt(m) + 40.0;
    long long total = 0;
    for (uint32_t c = 0; c < (uint32_t)n_chunks; ++c) {
        const double u = philox_uniform(seed, call, c, kDiPoisson);
        double p = std::exp(-m), F = p;
        long long k = 0;
        while (u > F && k < cap) {
            ++k;
            p *= m / (double)k;
            F += p;
        }
        total += k;
    }
    return total;
}

int di_args(skb_flow *fl, const char *who, const skb_dynamic_instability *di, double dt, int n_in,
            const skb_fiber_params *params_in, const int32_t *binding_in, const int32_t *plus_pinned, int capacity,
            int *n_out, skb_fiber_params *params_out, int32_t *binding_out, double *v_growth_out, int32_t *origin_out,
            skb_dynamic_info *info) {
    if (!di || !n_out || !info)
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    if (fl->grp.member())
        return set_error(SKB_ERR_INVALID, "%s: a group member's window is sized for a fixed fiber set", who);
    if (n_in != fl->n_fibers)
        return set_error(SKB_ERR_INVALID, "%s: n_in = %d, the flow has %d fibers", who, n_in, fl->n_fibers);
    if (n_in > 0 && (!params_in || !binding_in || !plus_pinned))
        return set_error(SKB_ERR_INVALID, "%s: NULL per-fiber input", who);
    const DynamicInstability &D = fl->dyn;
    const int nb = fl->n_bodies;
    const bool sites = D.sites_set && (int)D.site_count.size() == nb;
    const long long n_sites = sites ? D.site_off[(size_t)nb] : 0;
    if (nb > 0 && !sites)
        return set_error(SKB_ERR_INVALID, "%s: no nucleation sites for the flow's %d bodies "
                                          "(skb_flow_set_nucleation_sites)", who, nb);
    if (n_sites > 0 && !fl->placed)
        return set_error(SKB_ERR_INVALID, "%s: the bodies were not placed (skb_flow_place_bodies)", who);
    if ((long long)capacity < (long long)n_in + n_sites)
        return set_error(SKB_ERR_INVALID, "%s: capacity = %d (n_in + the %lld sites needed)", who, capacity, n_sites);
    if (capacity > 0 && (!params_out || !binding_out || !v_growth_out || !origin_out))
        return set_error(SKB_ERR_INVALID, "%s: NULL output", who);
    for (int f = 0; f < n_in; ++f) {
        const int b = binding_in[2 * f], s = binding_in[2 * f + 1];
        if (b != -1 && (b < 0 || b >= nb || s < 0 || s >= D.site_count[(size_t)b]))
            return set_error(SKB_ERR_INVALID, "%s: fiber %d is bound to (%d, %d), outside the sites", who, f, b, s);
        if (plus_pinned[f] != 0 && plus_pinned[f] != 1)
            return set_error(SKB_ERR_INVALID, "%s: plus_pinned[%d] = %d (must be 0 or 1)", who, f, plus_pinned[f]);
    }
    if (di->n_nodes == 0)
        return SKB_OK;
    if (!(dt > 0) || !std::isfinite(dt))
        return set_error(SKB_ERR_INVALID, "%s: dt = %g (must be finite and > 0)", who, dt);
    const double rates[6] = {di->v_growth, di->f_catastrophe, di->v_grow_collision_scale,
                             di->f_catastrophe_collision_scale, di->nucleation_rate, di->bending_rigidity};
    for (double v : rates)
        if (!(v >= 0) || !std::isfinite(v))
            return set_error(SKB_ERR_INVALID, "%s: a rate, scale or bending rigidity is %g (must be finite and >= 0)",
                             who, v);
    if (!(di->radius > 0) || !std::isfinite(di->radius) || !(di->min_length > 0) || !std::isfinite(di->min_length))
        return set_error(SKB_ERR_INVALID, "%s: radius = %g, min_length = %g (both must be finite and > 0)", who,
                         di->radius, di->min_length);
    if (!fl->ops.buildable(di->n_nodes))
        return set_error(SKB_ERR_INVALID, "%s: di.n_nodes = %d (must be in [%d, %d] with skb_flow_set_fiber_class and "
                                          "_class_derivatives)", who, di->n_nodes, FiberOps::build_min_nodes(),
                         FiberOps::build_max_nodes());
    return SKB_OK;
}

// the model itself, after di_args: the catastrophe and growth on the device, the count and picks on the host, the new
// block on the device and its install
int di_run(skb_flow *fl, const skb_dynamic_instability *di, double dt, uint64_t seed, uint64_t call, int n_in,
           const skb_fiber_params *params_in, const int32_t *binding_in, const int32_t *plus_pinned, int *n_out,
           skb_fiber_params *params_out, int32_t *binding_out, double *v_growth_out, int32_t *origin_out,
           skb_dynamic_info *info) {
    DynamicInstability &D = fl->dyn;
    const cudaStream_t st = fl->stream;
    const int nb = fl->n_bodies;
    const long long n_sites = nb > 0 ? D.site_off[(size_t)nb] : 0;

    // ---- per fiber: catastrophe, growth, occupancy; the survivor scan; one read-back ----
    DiRates r;
    r.thr[0] = std::exp(-dt * di->f_catastrophe);
    r.thr[1] = std::exp(-dt * (di->f_catastrophe * di->f_catastrophe_collision_scale));
    r.v[0] = di->v_growth;
    r.v[1] = di->v_growth * di->v_grow_collision_scale;
    r.dt = dt;
    r.seed = seed;
    r.call = call;
    std::vector<int2> fib((size_t)n_in);
    for (int f = 0; f < n_in; ++f) {
        const int b = binding_in[2 * f];
        fib[(size_t)f] = make_int2(b >= 0 ? (int)(D.site_off[(size_t)b] + binding_in[2 * f + 1]) : -1, plus_pinned[f]);
    }
    const size_t n_state = sizeof(DiCounts) + (size_t)n_in + (size_t)n_sites;
    SKB_TRY(D.counts.ensure(n_state));
    SKB_TRY(D.fib.ensure((size_t)n_in * sizeof(int2) + 8));
    SKB_TRY(D.len_new.ensure((size_t)n_in * 8 + 8));
    SKB_TRY(D.src.ensure((size_t)n_in * 4 + 8));
    SKB_TRY(D.dst_off.ensure((size_t)n_in * 8 + 8));
    if (n_state > D.h_cap) {
        D.h_counts.reset();
        D.h_cap = 0;
        CUDA_TRY(cudaMallocHost((void **)D.h_counts.out(), n_state));
        D.h_cap = n_state;
    }
    DiCounts *d_counts = (DiCounts *)D.counts.ptr;
    unsigned char *d_keep = (unsigned char *)D.counts.ptr + sizeof(DiCounts), *d_occ = d_keep + n_in;
    CUDA_TRY(cudaMemsetAsync(D.counts.ptr, 0, n_state, st));
    if (n_in > 0) {
        CUDA_TRY(cudaMemcpyAsync(D.fib.ptr, fib.data(), fib.size() * sizeof(int2), cudaMemcpyHostToDevice, st));
        di_decide_kernel<<<(n_in + kDiThreads - 1) / kDiThreads, kDiThreads, 0, st>>>(
            n_in, (const int2 *)D.fib.ptr, (const double *)fl->fiber_length.ptr, r, d_keep, (double *)D.len_new.ptr,
            d_occ, d_counts);
        CUDA_TRY(cudaGetLastError());
        di_scan_kernel<<<1, kDiScanThreads, 0, st>>>(n_in, d_keep, (const long long *)fl->fiber_offset.ptr,
                                                     (int *)D.src.ptr, (long long *)D.dst_off.ptr, d_counts);
        CUDA_TRY(cudaGetLastError());
        count_launch(2);
        fl->launches += 2;
    }
    CUDA_TRY(cudaMemcpyAsync(D.h_counts.get(), D.counts.ptr, n_state, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    DiCounts cnt;
    std::memcpy(&cnt, D.h_counts.get(), sizeof(cnt));
    const unsigned char *keep = (const unsigned char *)D.h_counts.get() + sizeof(DiCounts), *occ = keep + n_in;
    const int n_surv = (int)(cnt.scan >> kDiCountShift);
    const long long surv_nodes = (long long)(cnt.scan & kDiNodeMask);

    // ---- the nucleation count and the picks, on the host ----
    const double mu = dt * di->nucleation_rate * (double)(n_sites - cnt.n_bound);
    std::vector<int> inactive;
    for (long long i = 0; i < n_sites; ++i)
        if (!occ[i])
            inactive.push_back((int)i);
    const long long M = (long long)inactive.size();
    const int n_new = (int)std::min(poisson(mu, seed, call), M);
    std::vector<int2> picks((size_t)n_new);
    for (int k = 0; k < n_new; ++k) {
        const double u = philox_uniform(seed, call, (uint32_t)k, kDiPick);
        const long long j = k + std::min((long long)std::floor(u * (double)(M - k)), M - k - 1);
        std::swap(inactive[(size_t)k], inactive[(size_t)j]);
        const int flat = inactive[(size_t)k];
        const int b = (int)(std::upper_bound(D.site_off.begin(), D.site_off.end(), (long long)flat) -
                            D.site_off.begin()) - 1;
        picks[(size_t)k] = make_int2(flat, b);
    }

    // ---- the new block: survivors copied, nucleated fibers drawn; one download ----
    const int nf = n_surv + n_new;
    const long long n_fib = surv_nodes + (long long)n_new * di->n_nodes;
    std::vector<double> r_new(3 * (size_t)n_fib), len((size_t)nf);
    if (nf > 0) {
        std::vector<double> frames(12 * (size_t)nb);
        for (int b = 0; b < nb; ++b) {
            quaternion_rotation(fl->h_orient.data() + 4 * (size_t)b, &frames[12 * (size_t)b]);
            std::memcpy(&frames[12 * (size_t)b + 9], fl->h_centers.data() + 3 * (size_t)b, 24);
        }
        SKB_TRY(D.picks.ensure((size_t)n_new * sizeof(int2) + 8));
        SKB_TRY(D.frames.ensure(frames.size() * 8 + 8));
        SKB_TRY(D.r_new.ensure((size_t)n_fib * 24 + 8));
        SKB_TRY(D.len_out.ensure((size_t)nf * 8 + 8));
        if (n_new > 0) {
            CUDA_TRY(cudaMemcpyAsync(D.picks.ptr, picks.data(), picks.size() * sizeof(int2), cudaMemcpyHostToDevice,
                                     st));
            CUDA_TRY(cudaMemcpyAsync(D.frames.ptr, frames.data(), frames.size() * 8, cudaMemcpyHostToDevice, st));
        }
        const DiNew nw{di->n_nodes, di->min_length, surv_nodes};
        di_compact_kernel<<<nf, kDiCompactThreads, 0, st>>>(
            n_surv, (const int *)D.src.ptr, (const long long *)D.dst_off.ptr, (const long long *)fl->fiber_offset.ptr,
            (const double *)fl->r_fib.ptr, (const double *)D.len_new.ptr, (const int2 *)D.picks.ptr,
            (const double *)D.d_site_ref.ptr, (const double *)D.frames.ptr, nw, (double *)D.r_new.ptr,
            (double *)D.len_out.ptr);
        CUDA_TRY(cudaGetLastError());
        count_launch(1);
        fl->launches += 1;
        CUDA_TRY(cudaMemcpyAsync(r_new.data(), D.r_new.ptr, r_new.size() * 8, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(len.data(), D.len_out.ptr, len.size() * 8, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
    }

    // ---- the per-fiber tables of the new set ----
    std::vector<int> origin((size_t)nf), n_nodes((size_t)nf);
    for (int f = 0, j = 0; f < n_in; ++f)
        if (keep[f])
            origin[(size_t)j++] = f;
    for (int j = 0; j < nf; ++j) {
        if (j < n_surv) {
            const int f = origin[(size_t)j];
            params_out[j] = params_in[f];
            params_out[j].length_prev = fl->h_fiber_len[(size_t)f];
            binding_out[2 * j] = binding_in[2 * f];
            binding_out[2 * j + 1] = binding_in[2 * f + 1];
            v_growth_out[j] = r.v[plus_pinned[f]];
            n_nodes[(size_t)j] = fl->h_fiber_n[(size_t)f];
        } else {
            const int2 p = picks[(size_t)(j - n_surv)];
            origin[(size_t)j] = -1;
            params_out[j] = skb_fiber_params{di->min_length, di->bending_rigidity, di->radius, 500.0, 1.0, 1, 0};
            binding_out[2 * j] = p.y;
            binding_out[2 * j + 1] = (int)(p.x - D.site_off[(size_t)p.y]);
            v_growth_out[j] = 0.0;
            n_nodes[(size_t)j] = di->n_nodes;
        }
        origin_out[j] = origin[(size_t)j];
    }
    std::vector<int> hinged((size_t)nf, 0);
    const bool flags = fl->step_hinged.size() == (size_t)n_in;
    for (int j = 0; flags && j < n_surv; ++j)
        hinged[(size_t)j] = fl->step_hinged[(size_t)origin[(size_t)j]];
    *n_out = nf;
    info->removed = n_in - n_surv;
    info->nucleated = n_new;
    info->grown = n_surv;
    info->reserved = 0;
    info->mu = mu;

    // ---- install: the fibers, the shape's per-fiber flags, the step's flags, the workspace (only a CUDA error can
    // stop it half-way: every argument has passed its checks) ----
    SKB_TRY(skb_flow_set_fibers(fl, r_new.data(), n_nodes.data(), len.data(), nf));
    SKB_TRY(fl->shape.carry(origin.data(), n_in, nf, n_fib, fl->stream));
    if (flags)
        fl->step_hinged = std::move(hinged);
    else
        fl->step_hinged.clear();
    return fl->kry.blocks() > 0 ? skb_flow_set_gmres(fl, fl->kry.blocks()) : SKB_OK;
}

} // namespace

extern "C" {

int skb_flow_set_nucleation_sites(skb_flow *fl, const int *n_sites_per_body, const double *site_ref) {
    const char *who = "skb_flow_set_nucleation_sites";
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    const int nb = fl->n_bodies;
    if (nb > 0 && !n_sites_per_body)
        return set_error(SKB_ERR_INVALID, "%s: NULL count table for %d bodies", who, nb);
    std::vector<long long> off((size_t)nb + 1, 0);
    for (int b = 0; b < nb; ++b) {
        if (n_sites_per_body[b] < 0)
            return set_error(SKB_ERR_INVALID, "%s: body %d has %d sites", who, b, n_sites_per_body[b]);
        off[(size_t)b + 1] = off[(size_t)b] + n_sites_per_body[b];
    }
    const long long n = off[(size_t)nb];
    if (n > 0 && !site_ref)
        return set_error(SKB_ERR_INVALID, "%s: NULL site_ref", who);
    for (long long i = 0; i < n; ++i) {
        const double *s = site_ref + 3 * i;
        if (!std::isfinite(s[0]) || !std::isfinite(s[1]) || !std::isfinite(s[2]))
            return set_error(SKB_ERR_INVALID, "%s: site %lld is not finite", who, i);
        if (s[0] == 0.0 && s[1] == 0.0 && s[2] == 0.0)
            return set_error(SKB_ERR_INVALID, "%s: site %lld is at its body's centre (no direction)", who, i);
    }
    CUDA_TRY(cudaSetDevice(fl->dev));
    DynamicInstability &D = fl->dyn;
    D.sites_set = false;
    SKB_TRY(D.d_site_ref.ensure((size_t)n * 24 + 8));
    if (n > 0) {
        CUDA_TRY(cudaMemcpyAsync(D.d_site_ref.ptr, site_ref, (size_t)n * 24, cudaMemcpyHostToDevice, fl->stream));
        CUDA_TRY(cudaStreamSynchronize(fl->stream));
    }
    D.site_count.assign(n_sites_per_body, n_sites_per_body + nb);
    D.site_off = std::move(off);
    D.site_ref.assign(site_ref, site_ref + 3 * n);
    D.sites_set = true;
    return SKB_OK;
}

int skb_flow_dynamic_instability(skb_flow *fl, const skb_dynamic_instability *di, double dt, uint64_t seed,
                                 uint64_t counter, int n_in, const skb_fiber_params *params_in,
                                 const int32_t *binding_in, const int32_t *plus_pinned, int capacity, int *n_out,
                                 skb_fiber_params *params_out, int32_t *binding_out, double *v_growth_out,
                                 int32_t *origin_out, skb_dynamic_info *info) {
    const char *who = "skb_flow_dynamic_instability";
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    SKB_TRY(di_args(fl, who, di, dt, n_in, params_in, binding_in, plus_pinned, capacity, n_out, params_out,
                    binding_out, v_growth_out, origin_out, info));
    fl->launches = 0;
    std::memset(info, 0, sizeof(*info));
    if (di->n_nodes == 0) { // the reference's early return: nothing changes
        *n_out = n_in;
        for (int f = 0; f < n_in; ++f) {
            params_out[f] = params_in[f];
            binding_out[2 * f] = binding_in[2 * f];
            binding_out[2 * f + 1] = binding_in[2 * f + 1];
            v_growth_out[f] = 0.0;
            origin_out[f] = f;
        }
        return SKB_OK;
    }
    CUDA_TRY(cudaSetDevice(fl->dev));
    return di_run(fl, di, dt, seed, counter, n_in, params_in, binding_in, plus_pinned, n_out, params_out, binding_out,
                  v_growth_out, origin_out, info);
}

int skb_flow_step_flags(skb_flow *fl, int32_t *plus_hinged) {
    const char *who = "skb_flow_step_flags";
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    if (fl->step_hinged.size() != (size_t)fl->n_fibers || fl->step_hinged.empty() != (fl->n_fibers == 0))
        return set_error(SKB_ERR_INVALID, "%s: no step was installed for the flow's %d fibers", who, fl->n_fibers);
    if (fl->n_fibers > 0 && !plus_hinged)
        return set_error(SKB_ERR_INVALID, "%s: NULL plus_hinged", who);
    if (fl->n_fibers > 0)
        std::memcpy(plus_hinged, fl->step_hinged.data(), (size_t)fl->n_fibers * sizeof(int32_t));
    return SKB_OK;
}

} // extern "C"

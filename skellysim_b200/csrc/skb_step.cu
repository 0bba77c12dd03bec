// skb_step.cu -- System::step (system.cpp:482-492) of a single-device flow (include/skelly_b200_flow.h, skb_flow_step)
// and of a rank-per-GPU group member (skb_flow_group_step_device): the links, the fiber operators, the RHS and the
// solve of the existing calls, then the fiber step kernel (step_kernels.cuh), the bodies' step on the host and the
// installation of the new geometry.
#include "step_kernels.cuh"
#include "skb_internal.hpp"
#include "../../include/skelly_b200_flow.h"

#include <cmath>
#include <cstring>
#include <limits>
#include <vector>

using namespace skb;

static_assert(kStepMaxMembers == kMaxGroup, "StepGather holds one window per member");

__global__ void __launch_bounds__(kStepThreads)
    skb::group_fiber_step_kernel(const StepItem *__restrict__ items, const double *__restrict__ in,
                                 const double *__restrict__ class_mats, const int2 *__restrict__ class_ranges,
                                 const double *__restrict__ length, double *__restrict__ tension,
                                 const StepGather out) {
    fiber_step<true>(items, in, class_mats, class_ranges, length, tension, out);
}

int StepBuffers::size(int n_fibers, long long n_fib, int n_bodies) {
    n_fibers_ = -1; // a failed allocation leaves the buffers unsized
    SKB_TRY(items.ensure((size_t)n_fibers * sizeof(StepItem) + 8));
    SKB_TRY(err.ensure((size_t)n_fibers * 8 + 8));
    SKB_TRY(r_new.ensure((size_t)n_fib * 24 + 8));
    SKB_TRY(fext.ensure((size_t)n_fib * 24 + 8));
    SKB_TRY(tension.ensure((size_t)n_fib * 8 + 8));
    SKB_TRY(force.ensure((size_t)n_bodies * 24 + 8));
    SKB_TRY(torque.ensure((size_t)n_bodies * 24 + 8));
    const size_t n_check = 3 * (size_t)n_fib + 6 * (size_t)n_bodies + 1;
    if (n_check > check_cap_) {
        check.reset();
        check_cap_ = 0;
        CUDA_TRY(cudaMallocHost((void **)check.out(), n_check * 8));
        check_cap_ = n_check;
    }
    cudaFuncAttributes fa; // loads the kernels now: no lazy module load inside the step (a group member's peers may wait)
    CUDA_TRY(cudaFuncGetAttributes(&fa, fiber_step_kernel<true>));
    CUDA_TRY(cudaFuncGetAttributes(&fa, fiber_step_kernel<false>));
    CUDA_TRY(cudaFuncGetAttributes(&fa, group_fiber_step_kernel));
    n_fibers_ = n_fibers;
    n_fib_ = n_fib;
    n_bodies_ = n_bodies;
    return SKB_OK;
}

int skb::launch_fiber_step(const FlowState &s, const OwnFibers &own, const std::vector<StepItem> &items,
                           const double *d_in, bool from_solution, cudaStream_t st) {
    const int nf = own.count();
    if (nf == 0)
        return SKB_OK;
    StepBuffers &b = *s.buf;
    CUDA_TRY(cudaMemcpyAsync(b.items.ptr, items.data(), (size_t)nf * sizeof(StepItem), cudaMemcpyHostToDevice, st));
    const StepItem *it = (const StepItem *)b.items.ptr;
    const double *mats = s.ops->class_table();
    const int2 *ranges = s.ops->class_range_table();
    if (from_solution)
        fiber_step_kernel<true><<<nf, kStepThreads, 0, st>>>(it, d_in, mats, ranges, own.length + own.f0,
                                                             (double *)b.r_new.ptr, (double *)b.tension.ptr,
                                                             (double *)b.err.ptr);
    else
        fiber_step_kernel<false><<<nf, kStepThreads, 0, st>>>(it, d_in, mats, ranges, own.length + own.f0, nullptr,
                                                              nullptr, (double *)b.err.ptr);
    CUDA_TRY(cudaGetLastError());
    count_launch(1);
    return SKB_OK;
}

// BodyContainer::step / SphericalBody::step (body_container.cpp:48-61, body_spherical.cpp:13-35) of one body from its
// rows U, w, with two deviations (DESIGN.md §5): the body always moves to c + dt U, and the new quaternion is
// normalised.  phi = dt w; |phi| > 0: q_new = (cos |phi|/2, sin(|phi|/2) phi / |phi|) * q in Eigen's product order
void skb::body_step(const double *c, const double *q, const double *U, const double *w, double dt, double *c_new,
               double *q_new) {
    for (int k = 0; k < 3; ++k)
        c_new[k] = c[k] + U[k] * dt;
    const double phi[3] = {w[0] * dt, w[1] * dt, w[2] * dt};
    const double pn = std::sqrt(phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2]);
    if (!(pn != 0.0)) {
        std::memcpy(q_new, q, 4 * sizeof(double));
        return;
    }
    const double s = std::cos(0.5 * pn), sh = std::sin(0.5 * pn);
    const double p0 = sh * phi[0] / pn, p1 = sh * phi[1] / pn, p2 = sh * phi[2] / pn;
    const double r[4] = {s * q[0] - p0 * q[1] - p1 * q[2] - p2 * q[3], s * q[1] + p0 * q[0] + p1 * q[3] - p2 * q[2],
                         s * q[2] + p1 * q[0] + p2 * q[1] - p0 * q[3], s * q[3] + p2 * q[0] + p0 * q[2] - p1 * q[1]};
    const double nrm = std::sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3]);
    for (int k = 0; k < 4; ++k)
        q_new[k] = r[k] / nrm;
}

// the lab-frame nucleation site of every bound fiber (get_nucleation_site): c + R site_ref, R of the body's quaternion;
// 0 for a free fiber
void skb::nucleation_sites(int n_fibers, const int *body, const double *site_ref, const double *centers,
                      const double *orientations, std::vector<double> &sites) {
    sites.assign(3 * (size_t)n_fibers, 0.0);
    for (int f = 0; f < n_fibers; ++f) {
        const int b = body ? body[f] : -1;
        if (b < 0)
            continue;
        double R[9];
        quaternion_rotation(orientations + 4 * (size_t)b, R);
        const double *s = site_ref + 3 * (size_t)f, *c = centers + 3 * (size_t)b;
        for (int k = 0; k < 3; ++k)
            sites[3 * (size_t)f + k] = c[k] + (R[3 * k] * s[0] + R[3 * k + 1] * s[1] + R[3 * k + 2] * s[2]);
    }
}

void skb::body_rows(const int *n_nodes, int n_bodies, const double *x_bodies, std::vector<double> &uw) {
    uw.resize(6 * (size_t)n_bodies);
    long long off = 0;
    for (int b = 0; b < n_bodies; ++b) {
        off += 3LL * n_nodes[b];
        std::memcpy(&uw[6 * (size_t)b], x_bodies + off, 48);
        off += 6;
    }
}

bool skb::all_finite(const std::vector<double> &a) {
    for (double v : a)
        if (!std::isfinite(v))
            return false;
    return true;
}

// the flow's fiber error from the per-fiber maxima: their max and the first fiber attaining it (NaN wins)
void skb::reduce_errors(const std::vector<double> &err, double *max_error, int *worst) {
    *max_error = 0.0;
    *worst = -1;
    for (size_t f = 0; f < err.size(); ++f)
        if (*worst < 0 || err[f] > *max_error || (err[f] != err[f] && *max_error == *max_error)) {
            *max_error = err[f];
            *worst = (int)f;
        }
}

// the refusals of the step's scalar arguments, shared by skb_flow_step and skb_flow_group_step_device
static int step_scalar_args(const char *who, const skb_step_info *info, double dt, double eta, double tol,
                            int num_blocks, int max_iters) {
    if (!info)
        return set_error(SKB_ERR_INVALID, "%s: NULL info", who);
    if (!(dt > 0) || !std::isfinite(dt))
        return set_error(SKB_ERR_INVALID, "%s: dt = %g (must be finite and > 0)", who, dt);
    if (!(eta > 0) || !std::isfinite(eta))
        return set_error(SKB_ERR_INVALID, "%s: eta = %g (must be finite and > 0)", who, eta);
    if (!(tol > 0) || !std::isfinite(tol))
        return set_error(SKB_ERR_INVALID, "%s: tol = %g (must be finite and > 0)", who, tol);
    if (num_blocks < 1 || num_blocks > kMaxKrylov)
        return set_error(SKB_ERR_INVALID, "%s: num_blocks = %d (must be in [1, %d])", who, num_blocks, kMaxKrylov);
    if (max_iters < 0)
        return set_error(SKB_ERR_INVALID, "%s: max_iters = %d", who, max_iters);
    return SKB_OK;
}

extern "C" {

int skb_flow_step(skb_flow *fl, skb_dense *dn, const skb_fiber_params *params, const double *v_growth,
                  const double *force_scale, const double *f_external, const double *body_forces_torques,
                  const int *fiber_body, const double *site_ref, double dt, double eta, double tol, int num_blocks,
                  int max_iters, double *x, double *tension, skb_step_info *info) {
    const char *who = "skb_flow_step";
    // ---- every refusal, before any launch ----
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    SKB_TRY(step_scalar_args(who, info, dt, eta, tol, num_blocks, max_iters));
    SKB_TRY(flow_step_checks(fl, dn, who));
    const FlowState s = flow_state(fl);
    const int nf = s.fibers.count(), nb = s.n_bodies;
    const long long n_fib = s.fibers.nodes();
    if (nf > 0 && !params)
        return set_error(SKB_ERR_INVALID, "%s: NULL params", who);
    bool any_bound = false;
    for (int f = 0; f < nf; ++f) {
        const int b = fiber_body ? fiber_body[f] : -1;
        if (b < -1 || b >= nb)
            return set_error(SKB_ERR_INVALID, "%s: fiber %d is bound to body %d (the flow has %d bodies; -1 = free)",
                             who, f, b, nb);
        any_bound = any_bound || b >= 0;
    }
    if (any_bound && !site_ref)
        return set_error(SKB_ERR_INVALID, "%s: NULL site_ref with bound fibers", who);
    std::vector<double> sites, rigidity((size_t)nf);
    for (int f = 0; f < nf; ++f)
        rigidity[(size_t)f] = params[f].bending_rigidity;
    nucleation_sites(nf, fiber_body, site_ref, s.centers, s.orientations, sites);
    const cudaStream_t st = flow_stream(fl);
    SKB_TRY(s.bodies->set_links(s.fibers, *s.ops, nb, s.centers, fiber_body, sites.data(), rigidity.data(), st, true));
    SKB_TRY(s.ops->check_step(s.fibers, params, v_growth, force_scale));
    std::vector<StepItem> items;
    SKB_TRY(s.ops->step_items(s.fibers, items));
    for (long long i = 0; f_external && i < 3 * n_fib; ++i)
        if (!std::isfinite(f_external[i]))
            return set_error(SKB_ERR_INVALID, "%s: a non-finite external force", who);
    for (int i = 0; body_forces_torques && i < 6 * nb; ++i)
        if (!std::isfinite(body_forces_torques[i]))
            return set_error(SKB_ERR_INVALID, "%s: a non-finite external body force or torque", who);
    long long n = 0;
    std::array<long long, 6> key;
    SKB_TRY(flow_gmres_size(fl, who, &n, &key));
    Krylov &kry = flow_krylov(fl);
    if (n > 0 && (!kry.sized_for(n, key) || !s.buf->sized_for(nf, n_fib, nb)))
        return set_error(SKB_ERR_INVALID, "%s: call skb_flow_set_gmres for the current solution size (%lld)", who, n);
    if (n > 0 && num_blocks > kry.blocks())
        return set_error(SKB_ERR_INVALID, "%s: num_blocks = %d, skb_flow_set_gmres sized the workspace for %d", who,
                         num_blocks, kry.blocks());
    std::memset(info, 0, sizeof(*info));
    info->worst_fiber = -1;
    if (n == 0) { // the empty system: nothing moves
        info->solve.converged = 1;
        return SKB_OK;
    }

    // ---- System::step: the links, the operators, the RHS and the solve from the current placement ----
    StepBuffers &buf = *s.buf;
    SKB_TRY(skb_flow_set_fiber_links(fl, fiber_body, sites.data(), rigidity.data()));
    SKB_TRY(skb_flow_build_fiber_operators(fl, params, dt, eta));
    std::vector<double> F, T;
    if (body_forces_torques && nb > 0)
        split_forces_torques(body_forces_torques, nb, F, T);
    const bool fext = f_external && n_fib > 0;
    if (fext)
        CUDA_TRY(cudaMemcpyAsync(buf.fext.ptr, f_external, (size_t)n_fib * 24, cudaMemcpyHostToDevice, st));
    if (!F.empty()) {
        CUDA_TRY(cudaMemcpyAsync(buf.force.ptr, F.data(), F.size() * 8, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(buf.torque.ptr, T.data(), T.size() * 8, cudaMemcpyHostToDevice, st));
    }
    SKB_TRY(skb_flow_build_system_rhs_device(fl, params, v_growth, force_scale,
                                             fext ? (const double *)buf.fext.ptr : nullptr,
                                             F.empty() ? nullptr : (const double *)buf.force.ptr,
                                             F.empty() ? nullptr : (const double *)buf.torque.ptr, dt, eta,
                                             kry.stage_b(), st));
    SKB_TRY(skb_flow_solve_system_device(fl, dn, kry.stage_b(), eta, tol, num_blocks, max_iters, kry.stage_x(),
                                         &info->solve, nullptr, st));
    const double *d_x = kry.stage_x();

    // ---- the bodies' step from their rows [U; w], on the host: one copy of the body part, the rows picked here ----
    const long long body0 = 4 * n_fib + 3 * s.n_shell;
    std::vector<double> xb((size_t)(n - body0));
    if (nb > 0)
        CUDA_TRY(cudaMemcpyAsync(xb.data(), d_x + body0, xb.size() * 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    std::vector<double> uw, c_new(3 * (size_t)nb), q_new(4 * (size_t)nb);
    body_rows(s.bodies->frame_node_counts(), nb, xb.data(), uw);
    for (int b = 0; b < nb; ++b)
        body_step(s.centers + 3 * (size_t)b, s.orientations + 4 * (size_t)b, &uw[6 * (size_t)b],
                  &uw[6 * (size_t)b + 3], dt, &c_new[3 * (size_t)b], &q_new[4 * (size_t)b]);
    const bool bodies_finite = all_finite(uw);
    std::vector<double> sites_new;
    if (bodies_finite)
        nucleation_sites(nf, fiber_body, site_ref, c_new.data(), q_new.data(), sites_new);
    else
        sites_new.assign(3 * (size_t)nf, 0.0);

    // ---- the fibers' step, repin and error on the device; one download of the new positions ----
    for (int f = 0; f < nf; ++f) {
        StepItem &it = items[(size_t)f];
        it.bound = fiber_body && fiber_body[f] >= 0;
        std::memcpy(it.site, &sites_new[3 * (size_t)f], sizeof(it.site));
    }
    SKB_TRY(launch_fiber_step(s, s.fibers, items, d_x, true, st));
    std::vector<double> r_new(3 * (size_t)n_fib), err((size_t)nf);
    if (nf > 0) {
        CUDA_TRY(cudaMemcpyAsync(r_new.data(), buf.r_new.ptr, r_new.size() * 8, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(err.data(), buf.err.ptr, err.size() * 8, cudaMemcpyDeviceToHost, st));
        if (tension)
            CUDA_TRY(cudaMemcpyAsync(tension, buf.tension.ptr, (size_t)n_fib * 8, cudaMemcpyDeviceToHost, st));
    }
    if (x)
        CUDA_TRY(cudaMemcpyAsync(x, d_x, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (!bodies_finite || !all_finite(r_new)) { // not installed: the caller's restore has nothing to undo
        info->fiber_error = std::numeric_limits<double>::quiet_NaN();
        return set_error(SKB_ERR_STATE, "%s: the solution holds non-finite %s; the geometry is unchanged", who,
                         bodies_finite ? "fiber positions" : "body velocities");
    }
    reduce_errors(err, &info->fiber_error, &info->worst_fiber);

    // ---- install: the new positions through skb_flow_set_fibers (same node counts and lengths, so the partition and
    // the class table stay), the placement, the links at the new sites ----
    const std::vector<int> n_nodes(s.fibers.n, s.fibers.n + nf);
    const std::vector<double> length(s.length, s.length + nf);
    // (every argument below has passed its call's checks already: only a CUDA error can stop the install half-way)
    SKB_TRY(skb_flow_set_fibers(fl, r_new.data(), n_nodes.data(), length.data(), nf));
    if (nb > 0)
        SKB_TRY(skb_flow_place_bodies(fl, c_new.data(), q_new.data()));
    return skb_flow_set_fiber_links(fl, fiber_body, sites_new.data(), rigidity.data());
}

// skb_flow_step on a flow that is no group member, its device arguments through the host
static int step_not_member(skb_flow *fl, skb_dense *dn, const skb_fiber_params *params, const double *v_growth,
                           const double *force_scale, const double *d_f_external, const double *d_body_forces,
                           const double *d_body_torques, const int *fiber_body, const double *site_ref, double dt,
                           double eta, double tol, int num_blocks, int max_iters, double *d_x, double *d_tension,
                           skb_step_info *info, cudaStream_t st) {
    CUDA_TRY(cudaSetDevice(flow_device(fl)));
    const FlowState s = flow_state(fl);
    const long long n_fib = s.fibers.nodes();
    const int nb = s.n_bodies;
    std::vector<double> fext(d_f_external ? 3 * (size_t)n_fib : 0), F(3 * (size_t)nb, 0.0), T(3 * (size_t)nb, 0.0),
        ft;
    if (!fext.empty())
        CUDA_TRY(cudaMemcpyAsync(fext.data(), d_f_external, fext.size() * 8, cudaMemcpyDeviceToHost, st));
    if (nb > 0 && d_body_forces)
        CUDA_TRY(cudaMemcpyAsync(F.data(), d_body_forces, F.size() * 8, cudaMemcpyDeviceToHost, st));
    if (nb > 0 && d_body_torques)
        CUDA_TRY(cudaMemcpyAsync(T.data(), d_body_torques, T.size() * 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (nb > 0 && (d_body_forces || d_body_torques)) {
        ft.resize(6 * (size_t)nb);
        for (int b = 0; b < nb; ++b)
            for (int k = 0; k < 3; ++k) {
                ft[6 * (size_t)b + k] = F[3 * (size_t)b + k];
                ft[6 * (size_t)b + 3 + k] = T[3 * (size_t)b + k];
            }
    }
    const long long n = flow_whole_size(fl);
    std::vector<double> x(d_x ? (size_t)n : 0), tension(d_tension ? (size_t)n_fib : 0);
    const int rc = skb_flow_step(fl, dn, params, v_growth, force_scale, fext.empty() ? nullptr : fext.data(),
                                 ft.empty() ? nullptr : ft.data(), fiber_body, site_ref, dt, eta, tol, num_blocks,
                                 max_iters, d_x ? x.data() : nullptr, d_tension ? tension.data() : nullptr, info);
    if (rc != SKB_OK && rc != SKB_ERR_STATE)
        return rc;
    if (d_x && n > 0)
        CUDA_TRY(cudaMemcpyAsync(d_x, x.data(), (size_t)n * 8, cudaMemcpyHostToDevice, st));
    if (d_tension && n_fib > 0)
        CUDA_TRY(cudaMemcpyAsync(d_tension, tension.data(), (size_t)n_fib * 8, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return rc;
}

// count doubles of d (device, NULL: nothing to check) through the pinned host copy `h` on st: all finite?  A copy, not a
// launch, so a refusal on its result still comes before any launch
static int device_finite(const double *d, size_t count, double *h, cudaStream_t st, bool *finite) {
    *finite = true;
    if (count == 0 || !d)
        return SKB_OK;
    CUDA_TRY(cudaMemcpyAsync(h, d, count * 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    for (size_t i = 0; i < count && *finite; ++i)
        *finite = std::isfinite(h[i]);
    return SKB_OK;
}

// System::step on one rank per GPU: the composed local-vector calls, then two epochs of the group's own protocol --
// the body rows all-gathered through x_body, the fiber step fused with the all-gather of its results through r_step --
// and the same decision and the same complete geometry on every member
int skb_flow_group_step_device(skb_flow *fl, skb_dense *dn_spc, skb_dense *dn_minv, const skb_fiber_params *params,
                               const double *v_growth, const double *force_scale, const double *d_f_external,
                               const double *d_body_forces, const double *d_body_torques, const int *fiber_body,
                               const double *site_ref, double dt, double eta, double tol, int num_blocks,
                               int max_iters, double *d_x_local, double *d_tension, skb_step_info *info,
                               void *stream) {
    const char *who = "skb_flow_group_step_device";
    const cudaStream_t st = (cudaStream_t)stream;
    // ---- every refusal, before any launch ----
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    if (!flow_group(fl).member())
        return step_not_member(fl, dn_spc, params, v_growth, force_scale, d_f_external, d_body_forces, d_body_torques,
                               fiber_body, site_ref, dt, eta, tol, num_blocks, max_iters, d_x_local, d_tension, info,
                               st);
    SKB_TRY(step_scalar_args(who, info, dt, eta, tol, num_blocks, max_iters));
    OwnFibers own;
    long long n = 0;
    std::array<long long, 6> key;
    SKB_TRY(flow_group_step_checks(fl, dn_spc, dn_minv, who, own, &n, &key));
    const FlowState s = flow_state(fl);
    Group &G = flow_group(fl);
    const int nf = s.fibers.count(), nfo = own.count(), nb = s.n_bodies;
    const long long n_fib = s.fibers.nodes(), m = own.nodes(), n_sw = key[3] - key[2];
    if (nfo > 0 && !params)
        return set_error(SKB_ERR_INVALID, "%s: NULL params", who);
    bool any_bound = false;
    for (int f = 0; f < nfo; ++f) {
        const int b = fiber_body ? fiber_body[f] : -1;
        if (b < -1 || b >= nb)
            return set_error(SKB_ERR_INVALID, "%s: own fiber %d (fiber %d) is bound to body %d (the flow has %d "
                                              "bodies; -1 = free)", who, f, own.f0 + f, b, nb);
        any_bound = any_bound || b >= 0;
    }
    if (any_bound && !site_ref)
        return set_error(SKB_ERR_INVALID, "%s: NULL site_ref with bound fibers", who);
    std::vector<double> sites, rigidity((size_t)nfo);
    for (int f = 0; f < nfo; ++f)
        rigidity[(size_t)f] = params[f].bending_rigidity;
    nucleation_sites(nfo, fiber_body, site_ref, s.centers, s.orientations, sites);
    SKB_TRY(s.bodies->set_links(own, *s.ops, nb, s.centers, fiber_body, sites.data(), rigidity.data(), flow_stream(fl),
                                true));
    SKB_TRY(s.ops->check_step(own, params, v_growth, force_scale));
    std::vector<StepItem> items;
    SKB_TRY(s.ops->step_items(own, items));
    Krylov &kry = flow_krylov(fl);
    if (!kry.sized_for(n, key) || !s.buf->sized_for(nf, n_fib, nb))
        return set_error(SKB_ERR_INVALID, "%s: call skb_flow_set_gmres for the member's current target ranges", who);
    if (!s.ops->build_sized_for(own)) // (the build's buffers are sized only once every class it needs is set)
        return set_error(SKB_ERR_INVALID, "%s: call skb_flow_set_gmres after the fiber classes and their derivatives "
                                          "are set (it sizes the fiber build's buffers)", who);
    // the device inputs through the pinned copy skb_flow_set_gmres sized: 24 B per own node, 48 B per body
    double *h = s.buf->check.get();
    bool fin_f = true, fin_b = true, fin_t = true;
    SKB_TRY(device_finite(d_f_external, 3 * (size_t)m, h, st, &fin_f));
    if (!fin_f)
        return set_error(SKB_ERR_INVALID, "%s: a non-finite external force", who);
    if (nb > 0) {
        SKB_TRY(device_finite(d_body_forces, 3 * (size_t)nb, h, st, &fin_b));
        SKB_TRY(device_finite(d_body_torques, 3 * (size_t)nb, h, st, &fin_t));
    }
    if (!fin_b || !fin_t)
        return set_error(SKB_ERR_INVALID, "%s: a non-finite external body force or torque", who);
    if (num_blocks > kry.blocks())
        return set_error(SKB_ERR_INVALID, "%s: num_blocks = %d, skb_flow_set_gmres sized the workspace for %d", who,
                         num_blocks, kry.blocks());
    std::memset(info, 0, sizeof(*info));
    info->worst_fiber = -1;
    if (flow_whole_size(fl) == 0) { // the empty system, on every member alike: nothing moves
        info->solve.converged = 1;
        return SKB_OK;
    }

    // ---- System::step: the links, the operators (on the flow's stream, drained), the RHS and the solve on st ----
    StepBuffers &buf = *s.buf;
    SKB_TRY(skb_flow_group_set_fiber_links(fl, fiber_body, sites.data(), rigidity.data()));
    SKB_TRY(skb_flow_build_fiber_operators(fl, params, dt, eta));
    CUDA_TRY(cudaStreamSynchronize(flow_stream(fl)));
    SKB_TRY(skb_flow_group_build_system_rhs_device(fl, params, v_growth, force_scale, d_f_external, d_body_forces,
                                                   d_body_torques, dt, eta, kry.stage_b(), st));
    SKB_TRY(skb_flow_group_solve_system_device(fl, dn_spc, dn_minv, kry.stage_b(), eta, tol, num_blocks, max_iters,
                                               kry.stage_x(), &info->solve, nullptr, st));
    const double *d_x = kry.stage_x(); // [4 per own fiber node | 3 per own periphery row | own body rows]
    int *launches = flow_launches(fl); // the protocol's launches join the flow's count, as in the other member calls

    // ---- the body rows all-gathered (an epoch of its own: the rows phase), [U; w] of every body from the own window
    // (48 bytes per body), the bodies' step on the host: every member from the same bits ----
    std::vector<double> uw(6 * (size_t)nb), c_new(3 * (size_t)nb), q_new(4 * (size_t)nb);
    if (nb > 0) {
        SKB_TRY(G.begin());
        SKB_TRY(G.store_rows(d_x + 4 * m + 3 * n_sw, nullptr, 0, 0, flow_num_sms(fl), st, launches));
        SKB_TRY(G.rows_barrier(true, true, st, launches));
        const int *nodes = s.bodies->frame_node_counts();
        long long off = 0;
        for (int b = 0; b < nb; ++b) {
            off += 3LL * nodes[b];
            CUDA_TRY(cudaMemcpyAsync(&uw[6 * (size_t)b], G.x_body() + off, 48, cudaMemcpyDeviceToHost, st));
            off += 6;
        }
        CUDA_TRY(cudaStreamSynchronize(st));
    }
    for (int b = 0; b < nb; ++b)
        body_step(s.centers + 3 * (size_t)b, s.orientations + 4 * (size_t)b, &uw[6 * (size_t)b],
                  &uw[6 * (size_t)b + 3], dt, &c_new[3 * (size_t)b], &q_new[4 * (size_t)b]);
    const bool bodies_finite = all_finite(uw);
    std::vector<double> sites_new;
    if (bodies_finite)
        nucleation_sites(nfo, fiber_body, site_ref, c_new.data(), q_new.data(), sites_new);
    else
        sites_new.assign(3 * (size_t)nfo, 0.0);

    // ---- the own fibers' step, repin and error fused with the all-gather of the results into r_step of every window
    // (an epoch of its own, the rows phase again), then the complete positions and errors from the own window ----
    std::vector<double> r_new(3 * (size_t)n_fib), err((size_t)nf);
    if (nf > 0) {
        SKB_TRY(G.begin());
        if (nfo > 0) {
            for (int f = 0; f < nfo; ++f) {
                StepItem &it = items[(size_t)f];
                it.bound = fiber_body && fiber_body[f] >= 0;
                std::memcpy(it.site, &sites_new[3 * (size_t)f], sizeof(it.site));
            }
            CUDA_TRY(cudaMemcpyAsync(buf.items.ptr, items.data(), (size_t)nfo * sizeof(StepItem),
                                     cudaMemcpyHostToDevice, st));
            StepGather g;
            g.size = G.step_windows(g.r_step);
            g.n_fib = n_fib;
            g.node0 = own.off[own.f0];
            g.fiber0 = own.f0;
            group_fiber_step_kernel<<<nfo, kStepThreads, 0, st>>>((const StepItem *)buf.items.ptr, d_x,
                                                                  s.ops->class_table(), s.ops->class_range_table(),
                                                                  own.length + own.f0, (double *)buf.tension.ptr, g);
            CUDA_TRY(cudaGetLastError());
            count_launch(1);
            *launches += 1;
        }
        SKB_TRY(G.rows_barrier(true, true, st, launches));
        CUDA_TRY(cudaMemcpyAsync(r_new.data(), G.r_step(), r_new.size() * 8, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(err.data(), G.r_step() + 3 * n_fib, err.size() * 8, cudaMemcpyDeviceToHost, st));
        if (d_tension && m > 0)
            CUDA_TRY(cudaMemcpyAsync(d_tension, buf.tension.ptr, (size_t)m * 8, cudaMemcpyDeviceToDevice, st));
    }
    if (d_x_local && n > 0)
        CUDA_TRY(cudaMemcpyAsync(d_x_local, d_x, (size_t)n * 8, cudaMemcpyDeviceToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st)); // the downloads land before this member's next signal

    // ---- one decision, from the complete arrays every member holds alike ----
    if (!bodies_finite || !all_finite(r_new)) {
        info->fiber_error = std::numeric_limits<double>::quiet_NaN();
        return set_error(SKB_ERR_STATE, "%s: the solution holds non-finite %s; the geometry is unchanged", who,
                         bodies_finite ? "fiber positions" : "body velocities");
    }
    reduce_errors(err, &info->fiber_error, &info->worst_fiber);

    // ---- install the complete geometry (same counts: the window, the partition and every buffer stay) ----
    const std::vector<int> n_nodes(s.fibers.n, s.fibers.n + nf);
    const std::vector<double> length(s.length, s.length + nf);
    SKB_TRY(skb_flow_set_fibers(fl, r_new.data(), n_nodes.data(), length.data(), nf));
    if (nb > 0)
        SKB_TRY(skb_flow_group_place_bodies(fl, c_new.data(), q_new.data()));
    SKB_TRY(skb_flow_group_set_fiber_links(fl, fiber_body, sites_new.data(), rigidity.data()));
    CUDA_TRY(cudaStreamSynchronize(flow_stream(fl)));
    return SKB_OK;
}

int skb_flow_fiber_error(skb_flow *fl, double *max_error, double *per_fiber) {
    const char *who = "skb_flow_fiber_error";
    if (!fl || !max_error)
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    CUDA_TRY(cudaSetDevice(flow_device(fl)));
    const FlowState s = flow_state(fl);
    const int nf = s.fibers.count();
    std::vector<StepItem> items;
    SKB_TRY(s.ops->step_items(s.fibers, items));
    std::vector<double> err((size_t)nf);
    if (nf > 0) {
        const cudaStream_t st = flow_stream(fl);
        SKB_TRY(s.buf->items.ensure((size_t)nf * sizeof(StepItem)));
        SKB_TRY(s.buf->err.ensure((size_t)nf * 8));
        SKB_TRY(launch_fiber_step(s, s.fibers, items, s.fibers.r_fib, false, st));
        CUDA_TRY(cudaMemcpyAsync(err.data(), s.buf->err.ptr, (size_t)nf * 8, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
    }
    int worst = -1;
    reduce_errors(err, max_error, &worst);
    if (per_fiber)
        std::memcpy(per_fiber, err.data(), (size_t)nf * 8);
    return SKB_OK;
}

int skb_flow_get_placement(skb_flow *fl, double *centers, double *orientations) {
    const char *who = "skb_flow_get_placement";
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    const FlowState s = flow_state(fl);
    if (!s.placed)
        return set_error(SKB_ERR_INVALID, "%s: the bodies were not placed since skb_flow_set_bodies "
                                          "(skb_flow_place_bodies)", who);
    if (centers)
        std::memcpy(centers, s.centers, 24 * (size_t)s.n_bodies);
    if (orientations)
        std::memcpy(orientations, s.orientations, 32 * (size_t)s.n_bodies);
    return SKB_OK;
}

int skb_flow_get_fibers(skb_flow *fl, double *r_fib) {
    if (!fl)
        return set_error(SKB_ERR_INVALID, "skb_flow_get_fibers: NULL flow");
    const FlowState s = flow_state(fl);
    if (s.fibers.nodes() > 0 && !r_fib)
        return set_error(SKB_ERR_INVALID, "skb_flow_get_fibers: NULL argument");
    if (s.fibers.nodes() > 0)
        std::memcpy(r_fib, s.positions, (size_t)s.fibers.nodes() * 24);
    return SKB_OK;
}

} // extern "C"

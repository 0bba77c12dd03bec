// skb_step.cu -- System::step (system.cpp:482-492) of a single-device flow (include/skelly_b200_flow.h, skb_flow_step)
// and of a rank-per-GPU group member (skb_flow_group_step_device, which skb_mflow_step runs on every member): the
// links, the fiber operators, the RHS and the solve of the existing calls, then the fiber step kernel
// (step_kernels.cuh), the bodies' step on the host and the installation of the new geometry.
#include "step_kernels.cuh"
#include "skb_flow.hpp"

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

// fiber_step_kernel over the fibers `own` of fl on st (items from FiberOps::step_items; from_solution: d_in is their
// block of a solution, 4 per own node, new positions and tensions to fl->stepbuf; else d_in holds positions), errors to
// fl->stepbuf.err
static int launch_fiber_step(skb_flow *fl, const OwnFibers &own, const std::vector<StepItem> &items,
                             const double *d_in, bool from_solution, cudaStream_t st) {
    const int nf = own.count();
    if (nf == 0)
        return SKB_OK;
    StepBuffers &b = fl->stepbuf;
    CUDA_TRY(cudaMemcpyAsync(b.items.ptr, items.data(), (size_t)nf * sizeof(StepItem), cudaMemcpyHostToDevice, st));
    const StepItem *it = (const StepItem *)b.items.ptr;
    const double *mats = fl->ops.class_table();
    const int2 *ranges = fl->ops.class_range_table();
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
static void body_step(const double *c, const double *q, const double *U, const double *w, double dt, double *c_new,
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
static void nucleation_sites(int n_fibers, const int *body, const double *site_ref, const double *centers,
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

static bool all_finite(const std::vector<double> &a) {
    for (double v : a)
        if (!std::isfinite(v))
            return false;
    return true;
}

// the flow's fiber error from the per-fiber maxima: their max and the first fiber attaining it (NaN wins)
static void reduce_errors(const std::vector<double> &err, double *max_error, int *worst) {
    *max_error = 0.0;
    *worst = -1;
    for (size_t f = 0; f < err.size(); ++f)
        if (*worst < 0 || err[f] > *max_error || (err[f] != err[f] && *max_error == *max_error)) {
            *max_error = err[f];
            *worst = (int)f;
        }
}

// ---- the refusals ----------------------------------------------------------------------------------------------------
int skb::step_scalar_args(const char *who, const skb_step_info *info, double dt, double eta, double tol,
                          int num_blocks, int max_iters) {
    if (!info)
        return set_error(SKB_ERR_INVALID, "%s: NULL info", who);
    if (!(dt > 0) || !std::isfinite(dt))
        return set_error(SKB_ERR_INVALID, "%s: dt = %g (must be finite and > 0)", who, dt);
    if (!(eta > 0) || !std::isfinite(eta))
        return set_error(SKB_ERR_INVALID, "%s: eta = %g (must be finite and > 0)", who, eta);
    return solve_scalar_args(who, tol, num_blocks, max_iters);
}

int skb::step_fiber_args(const char *who, const skb_fiber_params *params, const int *fiber_body,
                         const double *site_ref, int f0, int nf, int nb) {
    if (nf > 0 && !params)
        return set_error(SKB_ERR_INVALID, "%s: NULL params", who);
    bool any_bound = false;
    for (int f = 0; f < nf; ++f) {
        const int b = fiber_body ? fiber_body[f] : -1;
        if (b < -1 || b >= nb)
            return set_error(SKB_ERR_INVALID, "%s: fiber %d is bound to body %d (the flow has %d bodies; -1 = free)",
                             who, f0 + f, b, nb);
        any_bound = any_bound || b >= 0;
    }
    if (any_bound && !site_ref)
        return set_error(SKB_ERR_INVALID, "%s: NULL site_ref with bound fibers", who);
    return SKB_OK;
}

int skb::step_host_inputs(const char *who, const double *f_external, long long n_fib,
                          const double *body_forces_torques, int nb) {
    for (long long i = 0; f_external && i < 3 * n_fib; ++i)
        if (!std::isfinite(f_external[i]))
            return set_error(SKB_ERR_INVALID, "%s: a non-finite external force", who);
    for (int i = 0; body_forces_torques && i < 6 * nb; ++i)
        if (!std::isfinite(body_forces_torques[i]))
            return set_error(SKB_ERR_INVALID, "%s: a non-finite external body force or torque", who);
    return SKB_OK;
}

// step_host_inputs for device inputs: the external forces of m fiber nodes and the forces and torques of the flow's
// bodies, read back into the pinned copy skb_flow_set_gmres sized (24 B per fiber node, 48 B per body) and scanned
// there.  Copies, not launches, so a refusal still comes before any launch
static int step_device_inputs(const char *who, skb_flow *fl, const double *d_f_external, long long m,
                              const double *d_body_forces, const double *d_body_torques, cudaStream_t st) {
    const size_t nb3 = fl->n_bodies > 0 ? 3 * (size_t)fl->n_bodies : 0;
    const double *d[3] = {d_f_external, d_body_forces, d_body_torques};
    const size_t count[3] = {3 * (size_t)m, nb3, nb3};
    double *h = fl->stepbuf.check.get();
    bool finite[3] = {true, true, true};
    for (int k = 0; k < 3; ++k) {
        if (!d[k] || count[k] == 0)
            continue;
        CUDA_TRY(cudaMemcpyAsync(h, d[k], count[k] * 8, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        for (size_t i = 0; i < count[k] && finite[k]; ++i)
            finite[k] = std::isfinite(h[i]);
    }
    if (!finite[0])
        return set_error(SKB_ERR_INVALID, "%s: a non-finite external force", who);
    if (!finite[1] || !finite[2])
        return set_error(SKB_ERR_INVALID, "%s: a non-finite external body force or torque", who);
    return SKB_OK;
}

// the refusals that concern the fibers the step advances (c.own): their arguments, their links at the current placement
// and their classes; c is left with their rigidity, current nucleation sites and items
static int own_fiber_checks(skb_flow *fl, const StepArgs &a, const char *who, StepCall &c) {
    const int nf = c.own.count();
    SKB_TRY(step_fiber_args(who, a.params, a.fiber_body, a.site_ref, c.own.f0, nf, fl->n_bodies));
    c.rigidity.resize((size_t)nf);
    for (int f = 0; f < nf; ++f)
        c.rigidity[(size_t)f] = a.params[f].bending_rigidity;
    nucleation_sites(nf, a.fiber_body, a.site_ref, fl->h_centers.data(), fl->h_orient.data(), c.sites);
    SKB_TRY(fl->bodies.set_links(c.own, fl->ops, fl->n_bodies, fl->h_centers.data(), a.fiber_body, c.sites.data(),
                                 c.rigidity.data(), fl->stream, true));
    SKB_TRY(fl->ops.check_step(c.own, a.params, a.v_growth, a.force_scale));
    return fl->ops.step_items(c.own, c.items);
}

// the step's buffers were sized for the flow as it is (skb_flow_set_gmres)
static bool step_sized(const skb_flow *fl) {
    return fl->stepbuf.sized_for(fl->n_fibers, fl->n_fib, fl->n_bodies);
}

// every refusal of skb_flow_step but its inputs' finiteness (they are on the host or on the device)
static int step_checks(skb_flow *fl, skb_dense *dn, const StepArgs &a, skb_step_info *info, const char *who,
                       StepCall &c) {
    SKB_TRY(step_scalar_args(who, info, a.dt, a.eta, a.tol, a.num_blocks, a.max_iters));
    if (fl->grp.member())
        return set_error(SKB_ERR_INVALID, "%s: a group member does not step (every member would need the others' new "
                                          "fiber positions); over several devices use skb_mflow", who);
    CUDA_TRY(cudaSetDevice(fl->dev));
    SKB_TRY(whole_targets(fl, who, ""));
    if (fl->n_shell > 0) {
        SKB_TRY(dense_rows(fl, dn, who, false));
        SKB_TRY(dense_rows(fl, dn, who, true));
    }
    SKB_TRY(system_ready(fl, who, kFlowCalls, true, true));
    c.own = all_fibers(fl);
    SKB_TRY(own_fiber_checks(fl, a, who, c));
    std::array<long long, 6> key;
    SKB_TRY(flow_gmres_size(fl, who, &c.n, &key));
    if (c.n > 0 && (!fl->kry.sized_for(c.n, key) || !step_sized(fl)))
        return set_error(SKB_ERR_INVALID, "%s: call skb_flow_set_gmres for the current solution size (%lld)", who, c.n);
    if (c.n > 0 && a.num_blocks > fl->kry.blocks())
        return set_error(SKB_ERR_INVALID, "%s: num_blocks = %d, skb_flow_set_gmres sized the workspace for %d", who,
                         a.num_blocks, fl->kry.blocks());
    return periphery_before_step(fl, who, a, c);
}

int skb::group_step_checks(skb_flow *fl, skb_dense *dn_spc, skb_dense *dn_minv, const StepArgs &a,
                           skb_step_info *info, const char *who, StepCall &c) {
    if (!fl->grp.member())
        return step_checks(fl, dn_spc, a, info, who, c);
    SKB_TRY(step_scalar_args(who, info, a.dt, a.eta, a.tol, a.num_blocks, a.max_iters));
    // its peers connected, its rows laid out for its target ranges, dn_spc / dn_minv its row blocks of the two
    // periphery operators, bodies placed with an inverse
    CUDA_TRY(cudaSetDevice(fl->dev));
    SKB_TRY(fl->grp.connected());
    SKB_TRY(own_fibers(fl, who, c.own)); // the target ranges resolved, whole fibers, the window's layout checked
    if (!fl->grp.rows_for(group_ranges(fl)))
        return set_error(SKB_ERR_INVALID, "%s: call skb_flow_group_set_body_frames / _set_body_operators after "
                                          "skb_flow_group_init and after every change of the target ranges", who);
    if (fl->sb > fl->sa) {
        SKB_TRY(dense_rows(fl, dn_spc, who, false));
        SKB_TRY(dense_rows(fl, dn_minv, who, true));
    }
    SKB_TRY(system_ready(fl, who, kGroupCalls, true, true));
    c.n = group_local_size(fl);
    SKB_TRY(own_fiber_checks(fl, a, who, c));
    if (!fl->kry.sized_for(c.n, group_ranges(fl)) || !step_sized(fl))
        return set_error(SKB_ERR_INVALID, "%s: call skb_flow_set_gmres for the member's current target ranges", who);
    if (!fl->ops.build_sized_for(c.own)) // (the build's buffers are sized only once every class it needs is set)
        return set_error(SKB_ERR_INVALID, "%s: call skb_flow_set_gmres after the fiber classes and their derivatives "
                                          "are set (it sizes the fiber build's buffers)", who);
    if (a.num_blocks > fl->kry.blocks())
        return set_error(SKB_ERR_INVALID, "%s: num_blocks = %d, skb_flow_set_gmres sized the workspace for %d", who,
                         a.num_blocks, fl->kry.blocks());
    return periphery_before_step(fl, who, a, c);
}

// ---- the pieces both runs share --------------------------------------------------------------------------------------
// uw = the rows [U; w] of every body (6 per body) from the body part of a solution on the device, 48 bytes per body
static int body_rows(const skb_flow *fl, const double *d_x_bodies, std::vector<double> &uw, cudaStream_t st) {
    uw.resize(6 * (size_t)fl->n_bodies);
    if (fl->n_bodies == 0)
        return SKB_OK;
    const int *nodes = fl->bodies.frame_node_counts();
    long long off = 0;
    for (int b = 0; b < fl->n_bodies; ++b) {
        off += 3LL * nodes[b];
        CUDA_TRY(cudaMemcpyAsync(&uw[6 * (size_t)b], d_x_bodies + off, 48, cudaMemcpyDeviceToHost, st));
        off += 6;
    }
    CUDA_TRY(cudaStreamSynchronize(st));
    return SKB_OK;
}

// the bodies' step from their rows uw, the new nucleation sites of the step's fibers (0 where a row is not finite: such
// a step is not installed) and their items' repin at them; false: a row is not finite
static bool advance_bodies(const skb_flow *fl, const StepArgs &a, const std::vector<double> &uw, StepCall &c,
                           std::vector<double> &c_new, std::vector<double> &q_new, std::vector<double> &sites_new) {
    c_new.resize(3 * (size_t)fl->n_bodies);
    q_new.resize(4 * (size_t)fl->n_bodies);
    for (int b = 0; b < fl->n_bodies; ++b)
        body_step(fl->h_centers.data() + 3 * (size_t)b, fl->h_orient.data() + 4 * (size_t)b, &uw[6 * (size_t)b],
                  &uw[6 * (size_t)b + 3], a.dt, &c_new[3 * (size_t)b], &q_new[4 * (size_t)b]);
    const bool finite = all_finite(uw);
    if (finite)
        nucleation_sites(c.own.count(), a.fiber_body, a.site_ref, c_new.data(), q_new.data(), sites_new);
    else
        sites_new.assign(3 * (size_t)c.own.count(), 0.0);
    for (size_t f = 0; f < c.items.size(); ++f) {
        c.items[f].bound = a.fiber_body && a.fiber_body[f] >= 0;
        std::memcpy(c.items[f].site, &sites_new[3 * f], sizeof(c.items[f].site));
    }
    return finite;
}

// one decision from the complete new positions and the bodies' rows: a non-finite solution is installed nowhere (the
// caller's restore has nothing to undo); else the fiber error
static int decide(const char *who, bool bodies_finite, const std::vector<double> &r_new,
                  const std::vector<double> &err, skb_step_info *info) {
    if (!bodies_finite || !all_finite(r_new)) {
        info->fiber_error = std::numeric_limits<double>::quiet_NaN();
        return set_error(SKB_ERR_STATE, "%s: the solution holds non-finite %s; the geometry is unchanged", who,
                         bodies_finite ? "fiber positions" : "body velocities");
    }
    reduce_errors(err, &info->fiber_error, &info->worst_fiber);
    return SKB_OK;
}

// ---- the two runs ----------------------------------------------------------------------------------------------------
// System::step of a single-device flow whose refusals have passed, on the flow's stream: d_f_external 3 per fiber node,
// d_body_forces / d_body_torques 3 per body (NULL: none); x / tension host or device memory (NULL: not wanted)
static int step_run(skb_flow *fl, skb_dense *dn, const StepArgs &a, StepCall &c, const double *d_f_external,
                    const double *d_body_forces, const double *d_body_torques, double *x, double *tension,
                    skb_step_info *info, const char *who) {
    std::memset(info, 0, sizeof(*info));
    info->worst_fiber = -1;
    if (c.n == 0) { // the empty system: nothing moves
        info->solve.converged = 1;
        return SKB_OK;
    }

    // ---- System::step: the links, the operators, the RHS and the solve from the current placement ----
    const int nf = fl->n_fibers, nb = fl->n_bodies;
    const long long n_fib = fl->n_fib;
    const cudaStream_t st = fl->stream;
    Krylov &kry = fl->kry;
    if (fl->shape.active() && n_fib > 0) { // f_external + the periphery's repulsion, into the step's own buffer
        SKB_TRY(periphery_add_force(fl, d_f_external, n_fib, (double *)fl->stepbuf.fext.ptr, st, &fl->launches));
        d_f_external = (const double *)fl->stepbuf.fext.ptr;
    }
    SKB_TRY(skb_flow_set_fiber_links(fl, a.fiber_body, c.sites.data(), c.rigidity.data()));
    SKB_TRY(skb_flow_build_fiber_operators(fl, c.params(a), a.dt, a.eta));
    SKB_TRY(skb_flow_build_system_rhs_device(fl, c.params(a), a.v_growth, a.force_scale,
                                             n_fib > 0 ? d_f_external : nullptr, nb > 0 ? d_body_forces : nullptr,
                                             nb > 0 ? d_body_torques : nullptr, a.dt, a.eta, kry.stage_b(), st));
    SKB_TRY(skb_flow_solve_system_device(fl, dn, kry.stage_b(), a.eta, a.tol, a.num_blocks, a.max_iters,
                                         kry.stage_x(), &info->solve, nullptr, st));
    const double *d_x = kry.stage_x();

    // ---- the bodies' step from their rows [U; w], on the host ----
    std::vector<double> uw, c_new, q_new, sites_new;
    SKB_TRY(body_rows(fl, d_x + 4 * n_fib + 3 * fl->n_shell, uw, st));
    const bool bodies_finite = advance_bodies(fl, a, uw, c, c_new, q_new, sites_new);

    // ---- the fibers' step, repin and error on the device; one download of the new positions ----
    SKB_TRY(launch_fiber_step(fl, all_fibers(fl), c.items, d_x, true, st));
    const StepBuffers &buf = fl->stepbuf;
    std::vector<double> r_new(3 * (size_t)n_fib), err((size_t)nf);
    if (nf > 0) {
        CUDA_TRY(cudaMemcpyAsync(r_new.data(), buf.r_new.ptr, r_new.size() * 8, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(err.data(), buf.err.ptr, err.size() * 8, cudaMemcpyDeviceToHost, st));
        if (tension)
            CUDA_TRY(cudaMemcpyAsync(tension, buf.tension.ptr, (size_t)n_fib * 8, cudaMemcpyDefault, st));
    }
    if (x)
        CUDA_TRY(cudaMemcpyAsync(x, d_x, (size_t)c.n * 8, cudaMemcpyDefault, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    SKB_TRY(decide(who, bodies_finite, r_new, err, info));

    // ---- install: the new positions through skb_flow_set_fibers (same node counts and lengths, so the partition and
    // the class table stay), the placement, the links at the new sites ----
    const std::vector<int> n_nodes(fl->h_fiber_n);
    const std::vector<double> length(fl->h_fiber_len);
    // (every argument below has passed its call's checks already: only a CUDA error can stop the install half-way)
    SKB_TRY(skb_flow_set_fibers(fl, r_new.data(), n_nodes.data(), length.data(), nf));
    if (nb > 0)
        SKB_TRY(skb_flow_place_bodies(fl, c_new.data(), q_new.data()));
    SKB_TRY(skb_flow_set_fiber_links(fl, a.fiber_body, sites_new.data(), c.rigidity.data()));
    // System::check_collision of the installed geometry, node 0 skipped on this step's is_minus_clamped()
    fl->shape.note_clamped(0, nf, c.params(a));
    // the bc_plus_ of the next dynamic instability's is_plus_pinned() (skb_flow_step_flags)
    fl->step_hinged.resize((size_t)nf);
    for (int f = 0; f < nf; ++f)
        fl->step_hinged[(size_t)f] = c.params(a)[f].plus_hinged;
    return periphery_collided(fl, &info->collided, st, &fl->launches);
}

// System::step on one rank per GPU: the composed local-vector calls, then two epochs of the group's own protocol --
// the body rows all-gathered through x_body, the fiber step fused with the all-gather of its results through r_step --
// and the same decision and the same complete geometry on every member
int skb::group_step_run(skb_flow *fl, skb_dense *dn_spc, skb_dense *dn_minv, const StepArgs &a, StepCall &c,
                        const double *d_f_external, const double *d_body_forces, const double *d_body_torques,
                        double *x_local, double *tension, skb_step_info *info, const char *who, cudaStream_t st) {
    if (!fl->grp.member()) { // skb_flow_step's run, on the flow's stream once the caller's work on st is done
        CUDA_TRY(cudaStreamSynchronize(st));
        return step_run(fl, dn_spc, a, c, d_f_external, d_body_forces, d_body_torques, x_local, tension, info, who);
    }
    std::memset(info, 0, sizeof(*info));
    info->worst_fiber = -1;
    if (solution_size(fl) == 0) { // the empty system, on every member alike: nothing moves
        info->solve.converged = 1;
        return SKB_OK;
    }

    // ---- System::step: the links, the operators (on the flow's stream, drained), the RHS and the solve on st ----
    Group &G = fl->grp;
    Krylov &kry = fl->kry;
    const StepBuffers &buf = fl->stepbuf;
    const int nf = fl->n_fibers, nfo = c.own.count(), nb = fl->n_bodies;
    const long long n_fib = fl->n_fib, m = c.own.nodes();
    int *launches = &fl->launches; // the protocol's launches join the flow's count, as in the other member calls
    if (fl->shape.active() && m > 0) { // f_external + the periphery's repulsion of the own nodes
        SKB_TRY(periphery_add_force(fl, d_f_external, m, (double *)buf.fext.ptr, st, launches));
        d_f_external = (const double *)buf.fext.ptr;
    }
    SKB_TRY(skb_flow_group_set_fiber_links(fl, a.fiber_body, c.sites.data(), c.rigidity.data()));
    SKB_TRY(skb_flow_build_fiber_operators(fl, c.params(a), a.dt, a.eta));
    CUDA_TRY(cudaStreamSynchronize(fl->stream));
    SKB_TRY(skb_flow_group_build_system_rhs_device(fl, c.params(a), a.v_growth, a.force_scale, d_f_external,
                                                   d_body_forces, d_body_torques, a.dt, a.eta, kry.stage_b(), st));
    SKB_TRY(skb_flow_group_solve_system_device(fl, dn_spc, dn_minv, kry.stage_b(), a.eta, a.tol, a.num_blocks,
                                               a.max_iters, kry.stage_x(), &info->solve, nullptr, st));
    const double *d_x = kry.stage_x(); // [4 per own fiber node | 3 per own periphery row | own body rows]

    // ---- the body rows all-gathered (an epoch of its own: the rows phase), [U; w] of every body from the own window,
    // the bodies' step on the host: every member from the same bits ----
    std::vector<double> uw, c_new, q_new, sites_new;
    if (nb > 0) {
        SKB_TRY(G.begin());
        SKB_TRY(G.store_rows(d_x + c.n - G.body_rows(), nullptr, 0, 0, fl->fib[1].info.num_sms, st,
                             launches));
        SKB_TRY(G.rows_barrier(true, true, st, launches));
        SKB_TRY(body_rows(fl, G.x_body(), uw, st));
    }
    const bool bodies_finite = advance_bodies(fl, a, uw, c, c_new, q_new, sites_new);

    // ---- the own fibers' step, repin and error fused with the all-gather of the results into r_step of every window
    // (an epoch of its own, the rows phase again), then the complete positions and errors from the own window ----
    // with a periphery shape, each own fiber's minus_clamped travels with its error: every member's collision test
    // then skips node 0 of the same fibers, and all of them return the same `collided` without another exchange
    const bool shape = fl->shape.active();
    std::vector<double> r_new(3 * (size_t)n_fib), err((size_t)nf), clamped(shape ? (size_t)nf : 0);
    if (nf > 0) {
        SKB_TRY(G.begin());
        if (nfo > 0) {
            CUDA_TRY(cudaMemcpyAsync(buf.items.ptr, c.items.data(), (size_t)nfo * sizeof(StepItem),
                                     cudaMemcpyHostToDevice, st));
            if (shape)
                SKB_TRY(fl->shape.upload_clamped(c.own.f0, nfo, c.params(a), st));
            StepGather g;
            g.size = G.step_windows(g.r_step);
            g.n_fib = n_fib;
            g.node0 = c.own.off[c.own.f0];
            g.fiber0 = c.own.f0;
            g.n_fibers = nf;
            g.clamp = shape ? fl->shape.clamp_table() : nullptr;
            group_fiber_step_kernel<<<nfo, kStepThreads, 0, st>>>((const StepItem *)buf.items.ptr, d_x,
                                                                  fl->ops.class_table(), fl->ops.class_range_table(),
                                                                  c.own.length + c.own.f0, (double *)buf.tension.ptr,
                                                                  g);
            CUDA_TRY(cudaGetLastError());
            count_launch(1);
            *launches += 1;
        }
        SKB_TRY(G.rows_barrier(true, true, st, launches));
        CUDA_TRY(cudaMemcpyAsync(r_new.data(), G.r_step(), r_new.size() * 8, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(err.data(), G.r_step() + 3 * n_fib, err.size() * 8, cudaMemcpyDeviceToHost, st));
        if (shape)
            CUDA_TRY(cudaMemcpyAsync(clamped.data(), G.r_step() + 3 * n_fib + nf, clamped.size() * 8,
                                     cudaMemcpyDeviceToHost, st));
        if (tension && m > 0)
            CUDA_TRY(cudaMemcpyAsync(tension, buf.tension.ptr, (size_t)m * 8, cudaMemcpyDefault, st));
    }
    if (x_local && c.n > 0)
        CUDA_TRY(cudaMemcpyAsync(x_local, d_x, (size_t)c.n * 8, cudaMemcpyDefault, st));
    CUDA_TRY(cudaStreamSynchronize(st)); // the downloads land before this member's next signal

    // ---- one decision, from the complete arrays every member holds alike ----
    SKB_TRY(decide(who, bodies_finite, r_new, err, info));

    // ---- install the complete geometry (same counts: the window, the partition and every buffer stay) ----
    const std::vector<int> n_nodes(fl->h_fiber_n);
    const std::vector<double> length(fl->h_fiber_len);
    SKB_TRY(skb_flow_set_fibers(fl, r_new.data(), n_nodes.data(), length.data(), nf));
    if (nb > 0)
        SKB_TRY(skb_flow_group_place_bodies(fl, c_new.data(), q_new.data()));
    SKB_TRY(skb_flow_group_set_fiber_links(fl, a.fiber_body, sites_new.data(), c.rigidity.data()));
    CUDA_TRY(cudaStreamSynchronize(fl->stream));
    // System::check_collision of the complete geometry every member installed, with the all-gathered flags: the same
    // on every member
    fl->shape.note_clamped_all(clamped);
    return periphery_collided(fl, &info->collided, fl->stream, launches);
}

extern "C" {

int skb_flow_step(skb_flow *fl, skb_dense *dn, const skb_fiber_params *params, const double *v_growth,
                  const double *force_scale, const double *f_external, const double *body_forces_torques,
                  const int *fiber_body, const double *site_ref, double dt, double eta, double tol, int num_blocks,
                  int max_iters, double *x, double *tension, skb_step_info *info) {
    const char *who = "skb_flow_step";
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    const StepArgs a{params, v_growth, force_scale, fiber_body, site_ref, dt, eta, tol, num_blocks, max_iters};
    StepCall c;
    SKB_TRY(step_checks(fl, dn, a, info, who, c));
    const long long n_fib = fl->n_fib;
    const int nb = fl->n_bodies;
    SKB_TRY(step_host_inputs(who, f_external, n_fib, body_forces_torques, nb));
    // the inputs into the step's own buffers, on the stream the step runs on
    StepBuffers &buf = fl->stepbuf;
    const cudaStream_t st = fl->stream;
    const bool fext = f_external && n_fib > 0, ft = body_forces_torques && nb > 0;
    if (fext)
        CUDA_TRY(cudaMemcpyAsync(buf.fext.ptr, f_external, (size_t)n_fib * 24, cudaMemcpyHostToDevice, st));
    std::vector<double> F, T;
    if (ft) {
        split_forces_torques(body_forces_torques, nb, F, T);
        CUDA_TRY(cudaMemcpyAsync(buf.force.ptr, F.data(), F.size() * 8, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(buf.torque.ptr, T.data(), T.size() * 8, cudaMemcpyHostToDevice, st));
    }
    return step_run(fl, dn, a, c, fext ? (const double *)buf.fext.ptr : nullptr,
                    ft ? (const double *)buf.force.ptr : nullptr, ft ? (const double *)buf.torque.ptr : nullptr, x,
                    tension, info, who);
}

int skb_flow_group_step_device(skb_flow *fl, skb_dense *dn_spc, skb_dense *dn_minv, const skb_fiber_params *params,
                               const double *v_growth, const double *force_scale, const double *d_f_external,
                               const double *d_body_forces, const double *d_body_torques, const int *fiber_body,
                               const double *site_ref, double dt, double eta, double tol, int num_blocks,
                               int max_iters, double *d_x_local, double *d_tension, skb_step_info *info,
                               void *stream) {
    const char *who = "skb_flow_group_step_device";
    const cudaStream_t st = (cudaStream_t)stream;
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    const StepArgs a{params, v_growth, force_scale, fiber_body, site_ref, dt, eta, tol, num_blocks, max_iters};
    StepCall c;
    SKB_TRY(group_step_checks(fl, dn_spc, dn_minv, a, info, who, c));
    SKB_TRY(step_device_inputs(who, fl, d_f_external, c.own.nodes(), d_body_forces, d_body_torques, st));
    return group_step_run(fl, dn_spc, dn_minv, a, c, d_f_external, d_body_forces, d_body_torques, d_x_local, d_tension,
                          info, who, st);
}

int skb_flow_fiber_error(skb_flow *fl, double *max_error, double *per_fiber) {
    const char *who = "skb_flow_fiber_error";
    if (!fl || !max_error)
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    CUDA_TRY(cudaSetDevice(fl->dev));
    const OwnFibers all = all_fibers(fl);
    const int nf = all.count();
    std::vector<StepItem> items;
    SKB_TRY(fl->ops.step_items(all, items));
    std::vector<double> err((size_t)nf);
    if (nf > 0) {
        const cudaStream_t st = fl->stream;
        SKB_TRY(fl->stepbuf.items.ensure((size_t)nf * sizeof(StepItem)));
        SKB_TRY(fl->stepbuf.err.ensure((size_t)nf * 8));
        SKB_TRY(launch_fiber_step(fl, all, items, all.r_fib, false, st));
        CUDA_TRY(cudaMemcpyAsync(err.data(), fl->stepbuf.err.ptr, (size_t)nf * 8, cudaMemcpyDeviceToHost, st));
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
    if (fl->n_bodies > 0 && !fl->placed)
        return set_error(SKB_ERR_INVALID, "%s: the bodies were not placed since skb_flow_set_bodies "
                                          "(skb_flow_place_bodies)", who);
    if (centers)
        std::memcpy(centers, fl->h_centers.data(), 24 * (size_t)fl->n_bodies);
    if (orientations)
        std::memcpy(orientations, fl->h_orient.data(), 32 * (size_t)fl->n_bodies);
    return SKB_OK;
}

int skb_flow_get_fibers(skb_flow *fl, double *r_fib) {
    if (!fl)
        return set_error(SKB_ERR_INVALID, "skb_flow_get_fibers: NULL flow");
    if (fl->n_fib > 0 && !r_fib)
        return set_error(SKB_ERR_INVALID, "skb_flow_get_fibers: NULL argument");
    if (fl->n_fib > 0)
        std::memcpy(r_fib, fl->h_r_fib.data(), (size_t)fl->n_fib * 24);
    return SKB_OK;
}

} // extern "C"

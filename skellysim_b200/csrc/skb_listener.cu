// skb_listener.cu -- the listener's frame and its requests (include/skelly_b200_flow.h, listener.cpp:86-136): the frame
// from the caller's strengths (set_frame) or from the installed geometry and a step's solution (set_state, the unpacking
// of trajectory_reader.cpp:150-249 and the strengths of System::velocity_at_targets, system.cpp:339-352); the
// velocity field (System::velocity_at_targets with its body-interior replacement, system.cpp:330-384) and streamlines
// and vortex lines (streamline.cpp), every line advanced at once (listener_kernels.cuh).  The velocity of every
// evaluation is skb::velocity_dev, the sequence of skb_flow_velocity_at_targets, at device targets.
#include "listener_kernels.cuh"
#include "skb_flow.hpp"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

using namespace skb;

static int load_listener_kernels() {
    static bool loaded = false;
    if (loaded)
        return SKB_OK;
    cudaFuncAttributes fa;
    CUDA_TRY(cudaFuncGetAttributes(&fa, interior_replace_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, gradient_finish_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, listener_state_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, line_init_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, line_compact_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, line_stage_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, line_control_kernel));
    SKB_TRY(load_source_kernels());
    loaded = true;
    return SKB_OK;
}

static unsigned blocks(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

// the rigid table (per body [kind, r0, r1, r2, cx, cy, cz, U, omega]) from the caller's interior tests and the body
// centres, U and omega from body_velocities (6 per body) or zero (NULL: a later launch writes them); *n_interior: the
// bodies with an interior test.  Refuses a bad kind or radius
static int rigid_table(const skb_flow *fl, const char *who, const int32_t *body_kind, const double *body_radii,
                       const double *body_velocities, std::vector<double> &rigid, int *n_interior) {
    const int nb = fl->n_bodies;
    rigid.assign((size_t)nb * kRigidStride, 0.0);
    *n_interior = 0;
    for (int b = 0; b < nb; ++b) {
        const int kind = body_kind[b];
        if (kind < 0 || kind > 2)
            return set_error(SKB_ERR_INVALID, "%s: body_kind[%d] = %d (must be 0, 1 or 2)", who, b, kind);
        for (int c = 0; c < (kind == 2 ? 3 : kind); ++c)
            if (!(body_radii[3 * b + c] > 0) || !std::isfinite(body_radii[3 * b + c]))
                return set_error(SKB_ERR_INVALID, "%s: body_radii[%d] = %g (must be finite and > 0 for body %d's "
                                                  "interior test)", who, 3 * b + c, body_radii[3 * b + c], b);
        double *p = rigid.data() + (size_t)b * kRigidStride;
        p[0] = kind;
        for (int c = 0; c < 3; ++c) {
            p[1 + c] = body_radii[3 * b + c];
            p[4 + c] = fl->h_centers[3 * (size_t)b + c];
            if (body_velocities) {
                p[7 + c] = body_velocities[6 * (size_t)b + c];
                p[10 + c] = body_velocities[6 * (size_t)b + 3 + c];
            }
        }
        *n_interior += kind != 0;
    }
    return SKB_OK;
}

// the frame is complete on the flow's stream: it takes the flow's geometry version
int Listener::commit(skb_flow *fl, int n_interior, double eta) {
    CUDA_TRY(cudaStreamSynchronize(fl->stream));
    SKB_TRY(load_listener_kernels());
    n_interior_ = n_interior;
    eta_ = eta;
    version_ = fl->geom_version;
    set_ = true;
    return SKB_OK;
}

int Listener::set_frame(skb_flow *fl, const double *fib_forces, const double *shell_density,
                        const double *body_densities, const double *body_forces_torques, const double *body_velocities,
                        const int32_t *body_kind, const double *body_radii, double eta) {
    const char *who = "skb_flow_set_listener_frame";
    if (!(eta > 0) || !std::isfinite(eta))
        return set_error(SKB_ERR_INVALID, "%s: eta = %g (must be finite and > 0)", who, eta);
    if ((fl->n_fib > 0 && !fib_forces) || (fl->n_shell > 0 && !shell_density) || (fl->n_body > 0 && !body_densities) ||
        (fl->n_bodies > 0 && (!body_forces_torques || !body_velocities || !body_kind || !body_radii)))
        return set_error(SKB_ERR_INVALID, "%s: NULL input for a non-empty class", who);
    const int nb = fl->n_bodies;
    std::vector<double> rigid;
    int n_interior = 0;
    SKB_TRY(rigid_table(fl, who, body_kind, body_radii, body_velocities, rigid, &n_interior));
    CUDA_TRY(cudaSetDevice(fl->dev));
    set_ = false; // a failed upload leaves no frame
    std::vector<double> f, t;
    if (nb > 0)
        split_forces_torques(body_forces_torques, nb, f, t);
    SKB_TRY(upload(fl, ff_, fib_forces, (size_t)fl->n_fib * 3));
    SKB_TRY(upload(fl, sd_, shell_density, (size_t)fl->n_shell * 3));
    SKB_TRY(upload(fl, bd_, body_densities, (size_t)fl->n_body * 3));
    SKB_TRY(upload(fl, f_, f.data(), f.size()));
    SKB_TRY(upload(fl, t_, t.data(), t.size()));
    SKB_TRY(upload(fl, rigid_, rigid.data(), rigid.size()));
    return commit(fl, n_interior, eta);
}

static int copy_async(DevBuf &dst, const double *src, size_t n_doubles, cudaStream_t st) {
    if (n_doubles == 0)
        return SKB_OK;
    SKB_TRY(dst.ensure(n_doubles * 8));
    CUDA_TRY(cudaMemcpyAsync(dst.ptr, src, n_doubles * 8, cudaMemcpyDeviceToDevice, st));
    return SKB_OK;
}

int Listener::set_state(skb_flow *fl, const skb_fiber_params *params, double dt, double eta, const double *tension,
                        const double *x, const int32_t *body_kind, const double *body_radii, int periphery_interaction,
                        bool device, cudaStream_t st) {
    const char *who = device ? "skb_flow_set_listener_state_device" : "skb_flow_set_listener_state";
    set_ = false; // a refused or failed call leaves no frame
    if (fl->grp.member())
        return set_error(SKB_ERR_INVALID, "%s: a group member's flow (the listener is single-device)", who);
    if (!(dt > 0) || !std::isfinite(dt) || !(eta > 0) || !std::isfinite(eta))
        return set_error(SKB_ERR_INVALID, "%s: dt = %g, eta = %g (both must be finite and > 0)", who, dt, eta);
    const long long nf = fl->n_fib, ns = fl->n_shell;
    const int nb = fl->n_bodies;
    if ((fl->n_fibers > 0 && (!params || !tension)) || ((ns > 0 || nb > 0) && !x) ||
        (nb > 0 && (!body_kind || !body_radii)))
        return set_error(SKB_ERR_INVALID, "%s: NULL input for a non-empty class", who);
    std::vector<double> rigid;
    int n_interior = 0;
    SKB_TRY(rigid_table(fl, who, body_kind, body_radii, nullptr, rigid, &n_interior));
    CUDA_TRY(cudaSetDevice(fl->dev));
    SKB_TRY(whole_targets(fl, who, ""));
    OwnFibers own;
    SKB_TRY(own_fibers(fl, who, own));
    SKB_TRY(fl->ops.check_step(own, params, nullptr, nullptr)); // the build's refusals: params, class derivatives
    if (nb > 0 && !fl->bodies.has_operators())
        return set_error(SKB_ERR_INVALID, "%s: call skb_flow_set_body_operators (or skb_flow_set_body_frames and "
                                          "skb_flow_place_bodies) after skb_flow_set_bodies", who);
    if (nb > 0 && fl->n_fibers > 0 && !fl->bodies.has_links())
        return set_error(SKB_ERR_INVALID, "%s: call skb_flow_set_fiber_links for the current geometry (NULL body: no "
                                          "fiber is bound)", who);
    if (periphery_interaction && nf > 0) // (the repulsion acts on fiber nodes only)
        SKB_TRY(periphery_ready(fl, who));
    for (long long i = 0; !device && i < nf; ++i)
        if (!std::isfinite(tension[i]))
            return set_error(SKB_ERR_INVALID, "%s: tension[%lld] = %g is not finite", who, i, tension[i]);
    if (device)
        CUDA_TRY(cudaStreamSynchronize(st)); // the caller's x and tension are complete
    begin_stats(fl);
    fl->cur = fl->stream;
    const cudaStream_t fs = fl->stream;
    // device_ms and total_ms both span the whole call on the flow's stream: elapsed stream time, the host waits after
    // the build's stages and the periphery pass's flag read-back included -- not the kernels' time alone
    CUDA_TRY(cudaEventRecord(fl->evt0, fs));
    CUDA_TRY(cudaEventRecord(fl->ev0, fs));
    // fc.update_cache_variables at the installed positions (trajectory_reader.cpp:248): force_operator_ and xs_ are
    // all the frame reads, so the build leaves out the inverse (most of a full build's time)
    SKB_TRY(fl->ops.build(
        own, params, dt, eta, &fl->launches,
        [&](const FiberOps::Step &stage, const FiberOps::Step &launch) -> int {
            SKB_TRY(stage());
            SKB_TRY(launch());
            CUDA_TRY(cudaStreamSynchronize(fs));
            return SKB_OK;
        },
        false));
    // the solution's shell and body blocks and the tension on the device
    const size_t n_sb = (size_t)(3 * ns + (nb > 0 ? fl->bodies.solution_size() : 0));
    const double *d_tension = tension, *d_sb = x ? x + 4 * nf : nullptr;
    if (!device) {
        SKB_TRY(upload(fl, ten_, tension, (size_t)nf));
        SKB_TRY(upload(fl, sb_, d_sb, n_sb));
        d_tension = (const double *)ten_.ptr;
        d_sb = (const double *)sb_.ptr;
    }
    const double *d_x_bodies = d_sb ? d_sb + 3 * ns : nullptr;
    SKB_TRY(xf_.ensure((size_t)nf * 32 + 8));
    SKB_TRY(ff_.ensure((size_t)nf * 24 + 8));
    SKB_TRY(upload(fl, rigid_, rigid.data(), rigid.size()));
    if (fl->n_fibers + nb > 0) {
        listener_state_kernel<<<(unsigned)(fl->n_fibers + nb), kStateThreads, 0, fs>>>(
            (const long long *)fl->fiber_offset.ptr, fl->n_fibers, (const double *)fl->r_fib.ptr, d_tension,
            (double *)xf_.ptr, fl->bodies.items(), d_x_bodies, (double *)rigid_.ptr);
        SKB_TRY(launched(&fl->launches));
    }
    // f_on_fibers = fc.apply_fiber_force(sol_fibers) (+ fc.periphery_force(shell, fp))      system.cpp:339-341
    SKB_TRY(fl->ops.force((const double *)xf_.ptr, (double *)ff_.ptr, fs, &fl->launches));
    if (periphery_interaction && nf > 0)
        SKB_TRY(periphery_add_repulsion(fl, who, (double *)ff_.ptr, fs, &fl->launches));
    // calculate_link_conditions(sol_fibers, sol_bodies): the link forces and torques, and the densities   :349-350
    if (nb > 0) {
        const double *link = nullptr;
        SKB_TRY(fl->bodies.links(fl->ops, (const double *)fl->fiber_length.ptr, (const double *)xf_.ptr, d_x_bodies,
                                 &link, fs, &fl->launches));
        SKB_TRY(copy_async(bd_, fl->bodies.densities(), (size_t)fl->n_body * 3, fs));
        SKB_TRY(copy_async(f_, fl->bodies.forces(), (size_t)nb * 3, fs));
        SKB_TRY(copy_async(t_, fl->bodies.torques(), (size_t)nb * 3, fs));
    }
    SKB_TRY(copy_async(sd_, d_sb, (size_t)ns * 3, fs));
    CUDA_TRY(cudaEventRecord(fl->ev1, fs));
    CUDA_TRY(cudaEventRecord(fl->evt1, fs));
    SKB_TRY(commit(fl, n_interior, eta));
    return finish_stats(fl);
}

int Listener::current(const skb_flow *fl, const char *who) const {
    if (!set_)
        return set_error(SKB_ERR_STATE, "%s: no listener frame (skb_flow_set_listener_frame)", who);
    if (version_ != fl->geom_version)
        return set_error(SKB_ERR_STATE, "%s: the listener frame is stale: the geometry, the point sources or the "
                                        "background flow changed after it was set", who);
    return SKB_OK;
}

int Listener::take_targets(skb_flow *fl, const double *d_trg, long long n_trg) {
    for (Evaluator *e : {&fl->fib[0], &fl->shell[0], &fl->body[0]})
        SKB_TRY(e->set_targets(d_trg, n_trg, true, fl->stream));
    // evaluation points are never taken for the fiber nodes: the plain kernel, without a device check (and its host
    // wait) for the symmetric one; the plain kernel's sum is right whatever the targets are
    fl->fib[0].src[SKB_STOKESLET].sym.self_state = 0;
    // the host-target calls must upload their targets again (and not replay a graph captured with theirs)
    fl->tc_fib.invalidate();
    fl->tc_shell.invalidate();
    fl->tc_body.invalidate();
    return SKB_OK;
}

int Listener::eval(skb_flow *fl, const double *d_trg, long long n_trg, double *d_v) {
    SKB_TRY(take_targets(fl, d_trg, n_trg));
    SKB_TRY(velocity_dev(fl, d_trg, n_trg, (const double *)ff_.ptr, (const double *)sd_.ptr, (const double *)bd_.ptr,
                         (const double *)f_.ptr, (const double *)t_.ptr, eta_, d_v));
    if (n_interior_ == 0)
        return SKB_OK;
    interior_replace_kernel<<<blocks(n_trg, kLineThreads), kLineThreads, 0, fl->cur>>>(
        d_trg, n_trg, (const double *)rigid_.ptr, fl->n_bodies, d_v);
    return launched(&fl->launches);
}

int Listener::velocity(skb_flow *fl, const double *r_trg, long long n_trg, double *vel) {
    const char *who = "skb_flow_listener_velocity";
    if (n_trg < 0 || (n_trg > 0 && (!r_trg || !vel)))
        return set_error(SKB_ERR_INVALID, "%s: bad arguments", who);
    SKB_TRY(current(fl, who));
    begin_stats(fl);
    if (n_trg == 0)
        return SKB_OK;
    CUDA_TRY(cudaSetDevice(fl->dev));
    return host_frame(
        fl,
        [&]() -> int {
            SKB_TRY(upload(fl, trg_, r_trg, (size_t)n_trg * 3));
            return vel_.ensure((size_t)n_trg * 24);
        },
        [&] { return eval(fl, (const double *)trg_.ptr, n_trg, (double *)vel_.ptr); },
        [&] { return download(fl, vel, vel_, (size_t)n_trg * 3); });
}

int Listener::gradient(skb_flow *fl, const double *r_trg, long long n_trg, double *grad, double *pressure) {
    const char *who = "skb_flow_listener_gradient";
    if (n_trg < 0 || (n_trg > 0 && (!r_trg || !grad || !pressure)))
        return set_error(SKB_ERR_INVALID, "%s: bad arguments", who);
    SKB_TRY(current(fl, who));
    begin_stats(fl);
    if (n_trg == 0)
        return SKB_OK;
    CUDA_TRY(cudaSetDevice(fl->dev));
    const double *d_trg = nullptr;
    auto work = [&]() -> int {
        SKB_TRY(take_targets(fl, d_trg, n_trg));
        SKB_TRY(gradient_dev(fl, d_trg, n_trg, (const double *)ff_.ptr, (const double *)sd_.ptr,
                             (const double *)bd_.ptr, (const double *)f_.ptr, (const double *)t_.ptr, eta_,
                             (double *)g10_.ptr));
        gradient_finish_kernel<<<blocks(n_trg, kLineThreads), kLineThreads, 0, fl->cur>>>(
            d_trg, n_trg, (const double *)rigid_.ptr, fl->n_bodies, eta_, (const double *)g10_.ptr,
            (double *)grad_.ptr, (double *)p_.ptr);
        return launched(&fl->launches);
    };
    return host_frame(
        fl,
        [&]() -> int {
            SKB_TRY(upload(fl, trg_, r_trg, (size_t)n_trg * 3));
            d_trg = (const double *)trg_.ptr;
            SKB_TRY(g10_.ensure((size_t)n_trg * 80));
            SKB_TRY(grad_.ensure((size_t)n_trg * 72));
            return p_.ensure((size_t)n_trg * 8);
        },
        work,
        [&]() -> int {
            SKB_TRY(download(fl, grad, grad_, (size_t)n_trg * 9));
            return download(fl, pressure, p_, (size_t)n_trg);
        });
}

static int line_args(const char *who, int kind, const double *x0, int n_lines, const skb_line_request *req,
                     const void *x, const void *t, const void *val, const void *n_points, const void *status) {
    if (kind != SKB_STREAMLINE && kind != SKB_VORTEXLINE)
        return set_error(SKB_ERR_INVALID, "%s: kind = %d (must be SKB_STREAMLINE or SKB_VORTEXLINE)", who, kind);
    if (n_lines < 0 || n_lines > (1 << 26))
        return set_error(SKB_ERR_INVALID, "%s: n_lines = %d (must be in [0, 2^26])", who, n_lines);
    if (n_lines == 0)
        return SKB_OK;
    if (!x0 || !req || !x || !t || !val || !n_points || !status)
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    for (long long i = 0; i < 3LL * n_lines; ++i)
        if (!std::isfinite(x0[i]))
            return set_error(SKB_ERR_INVALID, "%s: seed %lld is not finite", who, i / 3);
    const double f[4] = {req->dt_init, req->t_final, req->abs_err, req->rel_err};
    for (double v : f)
        if (!std::isfinite(v))
            return set_error(SKB_ERR_INVALID, "%s: a non-finite request field", who);
    if (!(req->dt_init > 0) || req->t_final < 0 || req->abs_err < 0 || req->rel_err < 0)
        return set_error(SKB_ERR_INVALID, "%s: dt_init = %g must be > 0; t_final = %g, abs_err = %g and rel_err = %g "
                                          "must be >= 0", who, req->dt_init, req->t_final, req->abs_err, req->rel_err);
    if (req->max_points < 1)
        return set_error(SKB_ERR_INVALID, "%s: max_points = %d (must be >= 1)", who, req->max_points);
    return SKB_OK;
}

int Listener::lines(skb_flow *fl, int kind, const double *x0, int n_lines, const skb_line_request *req, double *x,
                    double *t, double *val, int32_t *n_points, int32_t *status) {
    const char *who = "skb_flow_listener_lines";
    SKB_TRY(line_args(who, kind, x0, n_lines, req, x, t, val, n_points, status));
    SKB_TRY(current(fl, who));
    begin_stats(fl);
    if (n_lines == 0)
        return SKB_OK;
    CUDA_TRY(cudaSetDevice(fl->dev));
    const int L = 2 * n_lines, mp = req->max_points, vortex = kind == SKB_VORTEXLINE;
    const size_t per = (size_t)L * mp;
    SKB_TRY(st_x_.ensure((size_t)L * 24));
    SKB_TRY(st_t_.ensure((size_t)L * 8));
    SKB_TRY(st_dt_.ensure((size_t)L * 8));
    SKB_TRY(st_k_.ensure((size_t)L * 18 * 8));
    SKB_TRY(st_int_.ensure((size_t)L * 4 * sizeof(int)));
    SKB_TRY(out_x_.ensure(per * 24));
    SKB_TRY(out_t_.ensure(per * 8));
    SKB_TRY(out_val_.ensure(per * 24));
    SKB_TRY(slots_.ensure((size_t)L * sizeof(int)));
    SKB_TRY(n_act_.ensure(sizeof(int)));
    SKB_TRY(trg_.ensure((size_t)L * line_points(vortex) * 24));
    SKB_TRY(vel_.ensure((size_t)L * line_points(vortex) * 24));
    if (!h_n_act_)
        CUDA_TRY(cudaMallocHost((void **)h_n_act_.out(), sizeof(double)));
    int *ints = (int *)st_int_.ptr;
    LineState s{(double *)st_x_.ptr, (double *)st_t_.ptr, (double *)st_dt_.ptr, (double *)st_k_.ptr,
                ints, ints + L, ints + 2 * L, ints + 3 * L,
                (double *)out_x_.ptr, (double *)out_t_.ptr, (double *)out_val_.ptr, (const int *)slots_.ptr};
    const LineParams p{req->t_final, req->abs_err, req->rel_err, mp, vortex};
    int *h_n = (int *)h_n_act_.get();
    std::vector<int> h_int((size_t)2 * L);
    std::vector<double> hx, ht, hv;
    int m = 0; // the most points of one line and direction
    const double *d_trg = (const double *)trg_.ptr;
    double *d_vel = (double *)vel_.ptr;
    // one attempt of every active line: six stages, each one flow evaluation of the compacted stage points; then the
    // step control, the compaction, and the active count back to the host to size the next attempt's launches
    auto work = [&]() -> int {
        line_init_kernel<<<blocks(L, kLineThreads), kLineThreads, 0, fl->stream>>>(s, d_trg, n_lines, req->dt_init,
                                                                                    req->back_integrate != 0);
        SKB_TRY(launched(&fl->launches));
        for (;;) {
            line_compact_kernel<<<1, kCompactThreads, 0, fl->stream>>>(s.status, L, (int *)slots_.ptr,
                                                                       (int *)n_act_.ptr);
            SKB_TRY(launched(&fl->launches));
            CUDA_TRY(cudaMemcpyAsync(h_n, n_act_.ptr, sizeof(int), cudaMemcpyDeviceToHost, fl->stream));
            CUDA_TRY(cudaStreamSynchronize(fl->stream));
            const int n_act = *h_n;
            if (n_act == 0)
                return SKB_OK;
            for (int stage = 1; stage <= 6; ++stage) {
                line_stage_kernel<<<blocks(n_act, kLineThreads), kLineThreads, 0, fl->stream>>>(s, p, stage, n_act,
                                                                                                 d_vel, (double *)d_trg);
                SKB_TRY(launched(&fl->launches));
                SKB_TRY(eval(fl, d_trg, (long long)n_act * line_points(vortex), d_vel));
            }
            line_control_kernel<<<blocks(n_act, kLineThreads), kLineThreads, 0, fl->stream>>>(s, p, n_act, d_vel);
            SKB_TRY(launched(&fl->launches));
        }
    };
    // the counts and exits, then the used part of every line's output in one strided copy per array
    auto down = [&]() -> int {
        CUDA_TRY(cudaMemcpyAsync(h_int.data(), ints, (size_t)2 * L * sizeof(int), cudaMemcpyDeviceToHost, fl->stream));
        CUDA_TRY(cudaStreamSynchronize(fl->stream));
        m = *std::max_element(h_int.begin() + L, h_int.end());
        hx.resize((size_t)L * m * 3);
        ht.resize((size_t)L * m);
        hv.resize((size_t)L * m * 3);
        if (m == 0)
            return SKB_OK;
        CUDA_TRY(cudaMemcpy2DAsync(hx.data(), (size_t)m * 24, out_x_.ptr, (size_t)mp * 24, (size_t)m * 24, L,
                                   cudaMemcpyDeviceToHost, fl->stream));
        CUDA_TRY(cudaMemcpy2DAsync(ht.data(), (size_t)m * 8, out_t_.ptr, (size_t)mp * 8, (size_t)m * 8, L,
                                   cudaMemcpyDeviceToHost, fl->stream));
        CUDA_TRY(cudaMemcpy2DAsync(hv.data(), (size_t)m * 24, out_val_.ptr, (size_t)mp * 24, (size_t)m * 24, L,
                                   cudaMemcpyDeviceToHost, fl->stream));
        return SKB_OK;
    };
    SKB_TRY(host_frame(fl, [&] { return upload(fl, trg_, x0, (size_t)n_lines * 3); }, work, down));
    // join_back_and_forward: the back points reversed without their copy of x0, then the forward points
    const size_t row = 2 * (size_t)mp - 1;
    for (int i = 0; i < n_lines; ++i) {
        const int lb = 2 * i, lf = 2 * i + 1, nb = h_int[L + lb], nf = h_int[L + lf];
        size_t o = (size_t)i * row;
        auto put = [&](int l, int q) {
            const size_t src = (size_t)l * m + q;
            std::memcpy(x + 3 * o, hx.data() + 3 * src, 24);
            std::memcpy(val + 3 * o, hv.data() + 3 * src, 24);
            t[o] = ht[src];
            ++o;
        };
        for (int q = nb - 1; q >= 1; --q)
            put(lb, q);
        for (int q = 0; q < nf; ++q)
            put(lf, q);
        n_points[i] = (int32_t)(o - (size_t)i * row);
        status[2 * i] = h_int[lb];
        status[2 * i + 1] = h_int[lf];
    }
    return SKB_OK;
}

extern "C" {

int skb_flow_set_listener_frame(skb_flow *fl, const double *fib_forces, const double *shell_density,
                                const double *body_densities, const double *body_forces_torques,
                                const double *body_velocities, const int32_t *body_kind, const double *body_radii,
                                double eta) {
    if (!fl)
        return set_error(SKB_ERR_INVALID, "skb_flow_set_listener_frame: NULL flow");
    return fl->listener.set_frame(fl, fib_forces, shell_density, body_densities, body_forces_torques, body_velocities,
                                  body_kind, body_radii, eta);
}

int skb_flow_set_listener_state(skb_flow *fl, const skb_fiber_params *params, double dt, double eta,
                                const double *tension, const double *x, const int32_t *body_kind,
                                const double *body_radii, int32_t periphery_interaction) {
    if (!fl)
        return set_error(SKB_ERR_INVALID, "skb_flow_set_listener_state: NULL flow");
    return fl->listener.set_state(fl, params, dt, eta, tension, x, body_kind, body_radii, periphery_interaction, false,
                                  nullptr);
}

int skb_flow_set_listener_state_device(skb_flow *fl, const skb_fiber_params *params, double dt, double eta,
                                       const double *d_tension, const double *d_x, const int32_t *body_kind,
                                       const double *body_radii, int32_t periphery_interaction, void *stream) {
    if (!fl)
        return set_error(SKB_ERR_INVALID, "skb_flow_set_listener_state_device: NULL flow");
    return fl->listener.set_state(fl, params, dt, eta, d_tension, d_x, body_kind, body_radii, periphery_interaction,
                                  true, (cudaStream_t)stream);
}

int skb_flow_listener_velocity(skb_flow *fl, const double *r_trg, int64_t n_trg, double *vel) {
    if (!fl)
        return set_error(SKB_ERR_INVALID, "skb_flow_listener_velocity: NULL flow");
    return fl->listener.velocity(fl, r_trg, n_trg, vel);
}

int skb_flow_listener_gradient(skb_flow *fl, const double *r_trg, int64_t n_trg, double *grad, double *pressure) {
    if (!fl)
        return set_error(SKB_ERR_INVALID, "skb_flow_listener_gradient: NULL flow");
    return fl->listener.gradient(fl, r_trg, n_trg, grad, pressure);
}

int skb_flow_listener_lines(skb_flow *fl, int kind, const double *x0, int32_t n_lines, const skb_line_request *req,
                            double *x, double *t, double *val, int32_t *n_points, int32_t *status) {
    if (!fl)
        return set_error(SKB_ERR_INVALID, "skb_flow_listener_lines: NULL flow");
    return fl->listener.lines(fl, kind, x0, n_lines, req, x, t, val, n_points, status);
}

} // extern "C"

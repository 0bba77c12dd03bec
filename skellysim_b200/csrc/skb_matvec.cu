// skb_matvec.cu -- the evaluations and the matvec of a flow (include/skelly_b200_flow.h): the FiberContainer /
// Periphery / BodyContainer flows of SkellySim at arbitrary targets, the point sources and the background flow, their
// sum at arbitrary targets (System::velocity_at_targets) with the CUDA-graph replay of small calls, the matvec target
// lists and matvec_core -- the hydrodynamic part of System::apply_matvec (src/core/system.cpp:284-316) -- and
// apply_matvec_core around it.  Built on the flow's evaluators (Evaluator, skb_runtime.cu); everything between the
// upload of the strengths and the download of the velocities stays on the device.  The flow object itself is
// skb_flow.cu.
#include "aux_kernels.cuh"
#include "skb_flow.hpp"

#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

using namespace skb;

namespace {
// reference defaults of the regularised helpers (include/kernels.hpp:38-46): reg = 5e-3, eps = 1e-5
constexpr double kReg = 5e-3;
constexpr double kEps = 1e-5;
} // namespace

// self term of the fibers (fcfd.cpp:203-210): d_vel rows [0, node_end - node_begin) are the fiber nodes
// [node_begin, node_end), the packed strengths are those of e's last Stokeslet evaluation
static int fiber_self_term(skb_flow *fl, const Evaluator &e, double eta, double *d_vel, long long node_begin,
                           long long node_end) {
    const SourceSet &s = e.src[SKB_STOKESLET];
    if (node_end <= node_begin || s.excl) // fused form: the pair kernels skipped every intra-fiber pair
        return SKB_OK;
    const size_t smem = (size_t)fl->max_fiber_nodes * 6 * sizeof(double);
    fiber_self_subtract_kernel<<<fl->n_fibers, 128, smem, fl->cur>>>(
        (const double *)fl->r_fib.ptr, s.f_cur, (const long long *)fl->fiber_offset.ptr, 1.0 / (8.0 * M_PI * eta),
        kReg * kReg, kEps, d_vel, node_begin, node_end);
    return launched(&fl->launches);
}

int skb::install_fiber_sources(skb_flow *fl) {
    const int max_n = fl->max_fiber_nodes, n_fibers = fl->n_fibers;
    if (max_n * 48 > 48 * 1024)
        CUDA_TRY(cudaFuncSetAttribute(fiber_self_subtract_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      max_n * 48));
    // trapezoid weights straight into both Stokeslet source sets
    for (int k = 0; k < 2; ++k) {
        SourceSet &s = fl->fib[k].src[SKB_STOKESLET];
        SKB_TRY(s.weights.ensure((size_t)fl->n_fib * 8));
        fiber_weights_kernel<<<n_fibers, 64, 0, fl->stream>>>((const long long *)fl->fiber_offset.ptr,
                                                              (const double *)fl->fiber_length.ptr, n_fibers,
                                                              (double *)s.weights.ptr);
        SKB_TRY(launched(&fl->launches));
        s.has_weights = true;
    }
    return SKB_OK;
}

// ---- device-side flows: the evaluator already has its targets and sources ---------------------------------------
// mode / d_forces: the caller's forces (kRaw) or already packed strengths (kPacked).
// subtract_self: the first (node_end - node_begin) targets are the fiber nodes [node_begin, node_end)
static int fibers_dev(skb_flow *fl, Evaluator &e, StrengthMode mode, const double *d_forces, double eta,
                      int subtract_self, double *d_vel, int accumulate, long long node_begin, long long node_end) {
    // (no fibers: zeros, or nothing to add, fiber_container_finite_difference.cpp:178-179)
    // weighted forces -> Stokeslet all-to-all, / eta  (fcfd.cpp:185-199, kernels.cpp:365)
    SKB_TRY(e.eval(SKB_STOKESLET, mode, d_forces, 0.0, d_vel, accumulate, fl->cur, &fl->launches, nullptr, 1.0 / eta));
    fl->pairs += fl->n_fib * e.n_trg;
    if (!subtract_self)
        return SKB_OK;
    if (!e.src[SKB_STOKESLET].excl && e.n_trg < node_end - node_begin)
        return set_error(SKB_ERR_INVALID, "fiber flow with subtract_self needs the fiber nodes as the first "
                                          "%lld targets (n_trg = %lld)", node_end - node_begin, e.n_trg);
    return fiber_self_term(fl, e, eta, d_vel, node_begin, node_end);
}

// mode / d_density: the caller's densities (kNormalDensity) or already packed sym6 strengths (kPacked)
static int periphery_dev(skb_flow *fl, Evaluator &e, StrengthMode mode, const double *d_density, double eta,
                         double *d_vel, int accumulate) {
    // (no periphery: zeros, or nothing to add, periphery.cpp:57-58)
    // f_dl = 2 eta n (x) rho formed on the device, stresslet, / eta  (periphery.cpp:68-74, kernels.cpp:358)
    SKB_TRY(e.eval(SKB_STRESSLET, mode, d_density, 2.0 * eta, d_vel, accumulate, fl->cur, &fl->launches, nullptr,
                   1.0 / eta));
    fl->pairs += fl->n_shell * e.n_trg;
    return SKB_OK;
}

static int bodies_dev(skb_flow *fl, Evaluator &e, const double *d_density, const double *d_force,
                      const double *d_torque, double eta, double *d_vel, int accumulate) {
    if (e.n_trg == 0)
        return SKB_OK;
    if (fl->n_bodies == 0) { // body_container.cpp:273-276
        if (!accumulate)
            CUDA_TRY(cudaMemsetAsync(d_vel, 0, (size_t)e.n_trg * 24, fl->cur));
        return SKB_OK;
    }
    // stresslet of the surface nodes (body_container.cpp:296-305)
    SKB_TRY(e.eval(SKB_STRESSLET, kNormalDensity, d_density, 2.0 * eta, d_vel, accumulate, fl->cur, &fl->launches,
                   nullptr, 1.0 / eta));
    // Stokeslet of the net forces at the centres (:327)
    SKB_TRY(e.eval(SKB_STOKESLET, kRaw, d_force, 0.0, d_vel, 1, fl->cur, &fl->launches, nullptr, 1.0 / eta));
    // rotlet of the net torques at the centres (:335, kernels.cpp:206-242)
    const int bs = 128;
    rotlet_add_kernel<<<(unsigned)((e.n_trg + bs - 1) / bs), bs, 0, fl->cur>>>(
        (const double *)fl->centers.ptr, d_torque, fl->n_bodies, (const double *)e.r_trg.ptr, e.n_trg,
        1.0 / (8.0 * M_PI * eta), kReg * kReg, kEps * kEps, d_vel);
    fl->pairs += (fl->n_body + 2 * (long long)fl->n_bodies) * e.n_trg;
    return launched(&fl->launches);
}

int skb::add_sources(skb_flow *fl, const double *d_trg, long long n_trg, double eta, double *d_v, cudaStream_t st) {
    const int bs = 128;
    const unsigned nblk = (unsigned)((n_trg + bs - 1) / bs);
    if (n_trg == 0)
        return SKB_OK;
    if (fl->n_points > 0) {
        oseen_contract_add_kernel<<<nblk, bs, 0, st>>>((const double *)fl->pt_pos.ptr, (const double *)fl->pt_force.ptr,
                                                       fl->n_points, d_trg, n_trg, 1.0 / (8.0 * M_PI * eta),
                                                       kReg * kReg, kEps, d_v);
        rotlet_add_kernel<<<nblk, bs, 0, st>>>((const double *)fl->pt_pos.ptr, (const double *)fl->pt_torque.ptr,
                                               fl->n_points, d_trg, n_trg, 1.0 / (8.0 * M_PI * eta), kReg * kReg,
                                               kEps * kEps, d_v);
        SKB_TRY(launched(&fl->launches, 2));
    }
    if (fl->has_background) {
        background_add_kernel<<<nblk, bs, 0, st>>>(d_trg, n_trg, fl->bg_comp[0], fl->bg_comp[1], fl->bg_comp[2],
                                                   fl->bg_scale[0], fl->bg_scale[1], fl->bg_scale[2],
                                                   fl->bg_uniform[0], fl->bg_uniform[1], fl->bg_uniform[2], d_v);
        SKB_TRY(launched(&fl->launches));
    }
    return SKB_OK;
}

int skb::velocity_dev(skb_flow *fl, const double *d_trg, long long n_trg, const double *d_ff, const double *d_sd,
                      const double *d_bd, const double *d_f, const double *d_t, double eta, double *d_v) {
    // fc_->flow(r_trg, f_on_fibers, eta, /*subtract_self=*/false) + bc_.flow + shell_->flow   system.cpp:355-359
    SKB_TRY(fibers_dev(fl, fl->fib[0], kRaw, d_ff, eta, 0, d_v, 0, 0, 0));
    SKB_TRY(bodies_dev(fl, fl->body[0], d_bd, d_f, d_t, eta, d_v, 1));
    SKB_TRY(periphery_dev(fl, fl->shell[0], kNormalDensity, d_sd, eta, d_v, 1));
    // + psc_.flow(r_trg, eta, time) + bs_.flow(r_trg, eta)                                  system.cpp:358-359
    return add_sources(fl, d_trg, n_trg, eta, d_v, fl->cur);
}

int skb::gradient_dev(skb_flow *fl, const double *d_trg, long long n_trg, const double *d_ff, const double *d_sd,
                      const double *d_bd, const double *d_f, const double *d_t, double eta, double *d_g) {
    if (n_trg == 0)
        return SKB_OK;
    cudaStream_t st = fl->cur;
    const double c = 1.0 / (8.0 * M_PI * eta);
    const int bs = 128;
    const unsigned nblk = (unsigned)((n_trg + bs - 1) / bs);
    CUDA_TRY(cudaMemsetAsync(d_g, 0, (size_t)n_trg * 80, st));
    // the sources of velocity_dev in its order: fibers, bodies (surface, centres' forces and torques), periphery
    Evaluator &ef = fl->fib[0], &eb = fl->body[0], &es = fl->shell[0];
    SKB_TRY(ef.gradient(SKB_STOKESLET, kRaw, d_ff, 0.0, d_g, st, &fl->launches, 1.0 / eta));
    fl->pairs += fl->n_fib * n_trg;
    if (fl->n_bodies > 0) {
        SKB_TRY(eb.gradient(SKB_STRESSLET, kNormalDensity, d_bd, 2.0 * eta, d_g, st, &fl->launches, 1.0 / eta));
        SKB_TRY(eb.gradient(SKB_STOKESLET, kRaw, d_f, 0.0, d_g, st, &fl->launches, 1.0 / eta));
        rotlet_grad_add_kernel<<<nblk, bs, 0, st>>>((const double *)fl->centers.ptr, d_t, fl->n_bodies, d_trg, n_trg,
                                                    c, kReg * kReg, kEps * kEps, d_g);
        SKB_TRY(launched(&fl->launches));
        fl->pairs += (fl->n_body + 2 * (long long)fl->n_bodies) * n_trg;
    }
    SKB_TRY(es.gradient(SKB_STRESSLET, kNormalDensity, d_sd, 2.0 * eta, d_g, st, &fl->launches, 1.0 / eta));
    fl->pairs += fl->n_shell * n_trg;
    if (fl->n_points > 0) {
        oseen_grad_add_kernel<<<nblk, bs, 0, st>>>((const double *)fl->pt_pos.ptr, (const double *)fl->pt_force.ptr,
                                                   fl->n_points, d_trg, n_trg, c, kReg * kReg, kEps, d_g);
        rotlet_grad_add_kernel<<<nblk, bs, 0, st>>>((const double *)fl->pt_pos.ptr, (const double *)fl->pt_torque.ptr,
                                                    fl->n_points, d_trg, n_trg, c, kReg * kReg, kEps * kEps, d_g);
        SKB_TRY(launched(&fl->launches, 2));
    }
    if (fl->has_background) {
        background_grad_add_kernel<<<nblk, bs, 0, st>>>(n_trg, fl->bg_comp[0], fl->bg_comp[1], fl->bg_comp[2],
                                                        fl->bg_scale[0], fl->bg_scale[1], fl->bg_scale[2], d_g);
        SKB_TRY(launched(&fl->launches));
    }
    return SKB_OK;
}

int skb::load_source_kernels() {
    cudaFuncAttributes fa;
    CUDA_TRY(cudaFuncGetAttributes(&fa, oseen_contract_add_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, rotlet_add_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, background_add_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, oseen_grad_add_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, rotlet_grad_add_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, background_grad_add_kernel));
    return SKB_OK;
}


static int set_targets_cached(skb_flow *fl, Evaluator &e, TargetCache &tc, const double *r_trg, long long n_trg) {
    if (tc.same(r_trg, n_trg) && e.n_trg == n_trg)
        return SKB_OK;
    SKB_TRY(e.set_targets(r_trg, n_trg, false, fl->stream));
    CUDA_TRY(cudaStreamSynchronize(fl->stream));
    tc.store(r_trg, n_trg);
    return SKB_OK;
}


// ---- CUDA-graph helpers ----------------------------------------------------------------------------------------
static constexpr size_t kGraphMaxBytes = 512 * 1024; // strengths + velocities of one call; beyond this the copies
                                                     // and kernels dwarf the launch gaps and the plain path is used
static unsigned long long mix_key(unsigned long long h, unsigned long long v) {
    h ^= v + 0x9e3779b97f4a7c15ULL + (h << 6) + (h >> 2);
    return h;
}
static unsigned long long dbl_bits(double x) {
    unsigned long long b;
    std::memcpy(&b, &x, 8);
    return b;
}
static int ensure_stage(skb_flow *fl, size_t n_doubles) {
    if (n_doubles <= fl->h_stage_cap)
        return SKB_OK;
    fl->h_stage_cap = 0;
    fl->g_matvec.reset(); // graphs hold the old staging addresses
    fl->g_vat.reset();
    CUDA_TRY(cudaMallocHost((void **)fl->h_stage.out(), (n_doubles + 64) * 8));
    fl->h_stage_cap = n_doubles + 64;
    return SKB_OK;
}

// every device address a captured sequence may bake in: a reallocation anywhere invalidates the graph.  The staging
// slots of x, the workspace, the geometry and the buffers of the evaluators `which`
static unsigned long long buffer_key(const skb_flow *fl, int which, const Transfers &x) {
    unsigned long long h = 0x1234567ULL;
    for (const std::vector<Transfer> *list : {&x.up, &x.down})
        for (const Transfer &t : *list)
            h = mix_key(h, (unsigned long long)(uintptr_t)t.dev);
    const DevBuf *bufs[] = {&fl->tmp, &fl->pt_pos, &fl->pt_force, &fl->pt_torque, &fl->centers, &fl->r_fib};
    for (const DevBuf *b : bufs)
        h = mix_key(h, (unsigned long long)(uintptr_t)b->ptr);
    for (const Evaluator *e : {&fl->fib[which], &fl->shell[which], &fl->body[which]}) {
        h = mix_key(h, (unsigned long long)(uintptr_t)e->r_trg.ptr);
        h = mix_key(h, (unsigned long long)(uintptr_t)e->partial.ptr);
        for (int k = 0; k < 2; ++k) {
            h = mix_key(h, (unsigned long long)(uintptr_t)e->src[k].f_packed.ptr);
            h = mix_key(h, (unsigned long long)(uintptr_t)e->src[k].r.ptr);
        }
    }
    return h;
}

// Run `body` (asynchronous work on fl->stream, fixed addresses only) either directly, as a capture followed by a
// replay, or as a replay of the cached graph.  First call with a key: direct (it also warms every buffer); second
// call with the same key: captured; afterwards: one cudaGraphLaunch per call.
template <class Body> static int run_graphed(skb_flow *fl, skb_flow::GraphSlot &slot, unsigned long long key, Body body) {
    if (slot.exec && slot.key == key) {
        CUDA_TRY(cudaGraphLaunch(slot.exec, fl->stream));
        count_launch(slot.launches);
        fl->launches = slot.launches;
        fl->pairs = slot.pairs;
        return SKB_OK;
    }
    if (slot.seen == key && fl->graphs_enabled) {
        slot.reset();
        cudaGraph_t graph = nullptr;
        cudaGraphExec_t exec = nullptr;
        const long long before = launch_count();
        CUDA_TRY(cudaStreamBeginCapture(fl->stream, cudaStreamCaptureModeThreadLocal));
        const int rc = body();
        cudaError_t e = cudaStreamEndCapture(fl->stream, &graph);
        count_launch((int)(before - launch_count())); // nothing was launched while capturing
        if (rc == SKB_OK && e == cudaSuccess && graph &&
            cudaGraphInstantiate(&exec, graph, nullptr, nullptr, 0) == cudaSuccess) {
            *slot.exec.out() = exec; // the slot takes only a successfully instantiated graph
            cudaGraphDestroy(graph);
            slot.key = key;
            slot.launches = fl->launches;
            slot.pairs = fl->pairs;
            CUDA_TRY(cudaGraphLaunch(slot.exec, fl->stream));
            count_launch(slot.launches);
            return SKB_OK;
        }
        if (graph)
            cudaGraphDestroy(graph);
        (void)cudaGetLastError();
        fl->graphs_enabled = false; // capture is not possible in this process: stay on the direct path
        fl->launches = 0;
        fl->pairs = 0;
    }
    slot.seen = key;
    return body();
}

// host_call of a launch-bound call.  When its copies are small enough (and graphs are on), the pinned mode: the
// caller's arrays are copied into the pinned staging, whose fixed host addresses a graph's memcpy nodes need, laid
// out as x's runs in order; the whole sequence, copies included, runs through run_graphed under `key` and the
// addresses it bakes in (the evaluators `which`), between the frame's events; then the outputs go to the caller
template <class Work>
static int replayable_call(skb_flow *fl, skb_flow::GraphSlot &slot, int which, unsigned long long key, Transfers &x,
                           Work work) {
    size_t n = 0;
    for (const std::vector<Transfer> *list : {&x.up, &x.down})
        for (const Transfer &t : *list)
            for (const Run &r : t.runs)
                n += (size_t)r.len;
    if (!fl->graphs_enabled || n * 8 > kGraphMaxBytes)
        return host_call(fl, x, work);
    SKB_TRY(ensure_stage(fl, n));
    const std::vector<Transfer> out = x.down; // the caller's arrays
    long long at = 0;
    for (std::vector<Transfer> *list : {&x.up, &x.down})
        for (Transfer &t : *list) {
            for (Run &r : t.runs) {
                if (list == &x.up && t.host && r.len)
                    std::memcpy(fl->h_stage + at, t.host + r.whole, (size_t)r.len * 8);
                r.whole = at;
                at += r.len;
            }
            if (t.host)
                t.host = fl->h_stage;
        }
    SKB_TRY(stage_slots(fl->slots, x));
    key = mix_key(key, buffer_key(fl, which, x));
    SKB_TRY(host_frame(fl, nothing, [&] {
        return run_graphed(fl, slot, key, [&]() -> int {
            SKB_TRY(issue(x.up, true, fl->stream));
            SKB_TRY(work((const Transfers &)x));
            return issue(x.down, false, fl->stream);
        });
    }, nothing));
    for (size_t i = 0; i < out.size(); ++i)
        for (size_t j = 0; j < out[i].runs.size(); ++j)
            if (out[i].host && out[i].runs[j].len)
                std::memcpy(out[i].host + out[i].runs[j].whole, fl->h_stage + x.down[i].runs[j].whole,
                            (size_t)out[i].runs[j].len * 8);
    return SKB_OK;
}

extern "C" {

int skb_flow_fibers(skb_flow *fl, const double *r_trg, int64_t n_trg, const double *fib_forces, double eta,
                    int subtract_self, double *vel) {
    if (!fl || n_trg < 0 || (n_trg > 0 && (!r_trg || !vel)) || (fl->n_fib > 0 && !fib_forces) || !(eta > 0))
        return set_error(SKB_ERR_INVALID, "skb_flow_fibers: bad arguments");
    CUDA_TRY(cudaSetDevice(fl->dev));
    begin_stats(fl);
    SKB_TRY(set_targets_cached(fl, fl->fib[0], fl->tc_fib, r_trg, n_trg));
    if (n_trg == 0)
        return SKB_OK;
    Transfers xfer{{up(fib_forces, 3 * fl->n_fib)}, {down(vel, 3 * n_trg)}};
    return host_call(fl, xfer, [&](const Transfers &io) {
        return fibers_dev(fl, fl->fib[0], kRaw, io.up[0].dev, eta, subtract_self, io.down[0].dev, 0, 0, fl->n_fib);
    });
}

int skb_flow_periphery(skb_flow *fl, const double *r_trg, int64_t n_trg, const double *density, double eta,
                       double *vel) {
    if (!fl || n_trg < 0 || (n_trg > 0 && (!r_trg || !vel)) || (fl->n_shell > 0 && !density) || !(eta > 0))
        return set_error(SKB_ERR_INVALID, "skb_flow_periphery: bad arguments");
    CUDA_TRY(cudaSetDevice(fl->dev));
    begin_stats(fl);
    SKB_TRY(set_targets_cached(fl, fl->shell[0], fl->tc_shell, r_trg, n_trg));
    if (n_trg == 0)
        return SKB_OK;
    Transfers xfer{{up(density, 3 * fl->n_shell)}, {down(vel, 3 * n_trg)}};
    return host_call(fl, xfer, [&](const Transfers &io) {
        return periphery_dev(fl, fl->shell[0], kNormalDensity, io.up[0].dev, eta, io.down[0].dev, 0);
    });
}

int skb_flow_bodies(skb_flow *fl, const double *r_trg, int64_t n_trg, const double *densities,
                    const double *forces_torques, double eta, double *vel) {
    if (!fl || n_trg < 0 || (n_trg > 0 && (!r_trg || !vel)) || (fl->n_body > 0 && !densities) ||
        (fl->n_bodies > 0 && !forces_torques) || !(eta > 0))
        return set_error(SKB_ERR_INVALID, "skb_flow_bodies: bad arguments");
    CUDA_TRY(cudaSetDevice(fl->dev));
    begin_stats(fl);
    SKB_TRY(set_targets_cached(fl, fl->body[0], fl->tc_body, r_trg, n_trg));
    if (n_trg == 0)
        return SKB_OK;
    std::vector<double> f, t;
    split_forces_torques(forces_torques, fl->n_bodies, f, t);
    Transfers xfer{{up(densities, 3 * fl->n_body), up(f.data(), f.size()), up(t.data(), t.size())},
                   {down(vel, 3 * n_trg)}};
    return host_call(fl, xfer, [&](const Transfers &io) {
        return bodies_dev(fl, fl->body[0], io.up[0].dev, io.up[1].dev, io.up[2].dev, eta, io.down[0].dev, 0);
    });
}


int skb_flow_velocity_at_targets(skb_flow *fl, const double *r_trg, int64_t n_trg, const double *fib_forces,
                                 const double *shell_density, const double *body_densities,
                                 const double *body_forces_torques, double eta, double *vel) {
    if (!fl || n_trg < 0 || (n_trg > 0 && (!r_trg || !vel)) || !(eta > 0))
        return set_error(SKB_ERR_INVALID, "skb_flow_velocity_at_targets: bad arguments");
    if ((fl->n_fib > 0 && !fib_forces) || (fl->n_shell > 0 && !shell_density) || (fl->n_body > 0 && !body_densities) ||
        (fl->n_bodies > 0 && !body_forces_torques))
        return set_error(SKB_ERR_INVALID, "skb_flow_velocity_at_targets: NULL input for a non-empty class");
    CUDA_TRY(cudaSetDevice(fl->dev));
    begin_stats(fl);
    // the three "arbitrary target" evaluators share one cached target list
    SKB_TRY(set_targets_cached(fl, fl->fib[0], fl->tc_fib, r_trg, n_trg));
    SKB_TRY(set_targets_cached(fl, fl->shell[0], fl->tc_shell, r_trg, n_trg));
    SKB_TRY(set_targets_cached(fl, fl->body[0], fl->tc_body, r_trg, n_trg));
    if (n_trg == 0)
        return SKB_OK;
    std::vector<double> f, t;
    if (fl->n_bodies > 0)
        split_forces_torques(body_forces_torques, fl->n_bodies, f, t);
    Transfers xfer{{up(fib_forces, 3 * fl->n_fib), up(shell_density, 3 * fl->n_shell),
                    up(body_densities, 3 * fl->n_body), up(f.data(), f.size()), up(t.data(), t.size())},
                   {down(vel, 3 * n_trg)}};
    // the listener / streamline integrator asks for 1-6 targets per call (streamline.cpp:11-35): launch-bound
    unsigned long long key = mix_key(fl->geom_version, (unsigned long long)n_trg);
    key = mix_key(key, dbl_bits(eta));
    // same count but different targets: the captured sequence assumed the old targets' relation to the sources
    key = mix_key(key, fl->tc_fib.version);
    key = mix_key(key, fl->tc_shell.version);
    key = mix_key(key, fl->tc_body.version);
    return replayable_call(fl, fl->g_vat, 0, key, xfer, [&](const Transfers &io) {
        return velocity_dev(fl, (const double *)fl->fib[0].r_trg.ptr, n_trg, io.up[0].dev, io.up[1].dev, io.up[2].dev,
                            io.up[3].dev, io.up[4].dev, eta, io.down[0].dev);
    });
}

} // extern "C"

int skb::prepare_matvec_targets(skb_flow *fl) {
    const long long nf = fl->n_fib, ns = fl->n_shell, nb = fl->n_body, n_all = nf + ns + nb;
    if (!fl->mv_dirty)
        return SKB_OK;
    auto clampi = [](long long x, long long lo, long long hi) { return std::min(std::max(x, lo), hi); };
    if (fl->use_ranges) {
        const long long f0 = clampi(fl->rq_f0, 0, fl->n_fibers), f1 = clampi(fl->rq_f1, f0, fl->n_fibers);
        fl->fa = fl->n_fibers ? fl->h_fiber_off[(size_t)f0] : 0;
        fl->fb = fl->n_fibers ? fl->h_fiber_off[(size_t)f1] : 0;
        fl->sa = clampi(fl->rq_s0, 0, ns);
        fl->sb = clampi(fl->rq_s1, fl->sa, ns);
        fl->ba = clampi(fl->rq_b0, 0, nb);
        fl->bb = clampi(fl->rq_b1, fl->ba, nb);
    } else {
        long long w0 = fl->win_begin, w1 = fl->win_end < 0 ? n_all : fl->win_end;
        w0 = clampi(w0, 0, n_all);
        w1 = clampi(w1, w0, n_all);
        fl->fa = clampi(w0, 0, nf);
        fl->fb = clampi(w1, 0, nf);
        fl->sa = clampi(w0 - nf, 0, ns);
        fl->sb = clampi(w1 - nf, 0, ns);
        fl->ba = clampi(w0 - nf - ns, 0, nb);
        fl->bb = clampi(w1 - nf - ns, 0, nb);
    }
    const long long n_fw = fl->fb - fl->fa, n_sw = fl->sb - fl->sa, n_bw = fl->bb - fl->ba;
    fl->n_win = n_fw + n_sw + n_bw;
    const bool grouped = fl->grp.member();
    if (grouped) {
        if (!fl->use_ranges)
            return set_error(SKB_ERR_STATE, "group member: call skb_flow_set_target_ranges (own fibers / periphery rows / "
                                            "body rows) before the first matvec");
        SKB_TRY(fl->grp.check_layout(nf, ns, nb, fl->n_bodies, fl->n_fibers));
    }
    // group: fiber rows through the symmetric block rows of this member (partial sums, pulled together afterwards)
    // when the self-interaction is big enough for that kernel; otherwise the member's own rows with the plain kernel
    const bool sym_partial = grouped && nf >= 2LL * sym_block_nodes();
    // fiber <-> periphery pairs in one pass (cross_kernels.cuh) when both classes are big enough to matter and the
    // symmetric kernel carries the fiber rows (so that the fiber evaluator's remaining targets are the body rows only)
    static const int cross_env = [] {
        const char *e = getenv("SKB_CROSS");
        return e ? atoi(e) : -1;
    }();
    const int cmode = fl->cross_mode >= 0 ? fl->cross_mode : cross_env;
    const bool sym_rows = grouped ? sym_partial
                                  : (fl->fa == 0 && fl->fb == nf && fl->sa == 0 && fl->sb == ns &&
                                     nf >= (cmode == 1 ? 2LL * sym_block_nodes() : 4096));
    const bool use_cross = cmode != 0 && sym_rows && n_fw > 0 && ns >= (cmode == 1 ? 1 : 256);
    fl->plan.grouped = grouped;
    fl->plan.cross = use_cross;
    fl->plan.fib_rows = sym_partial ? skb_flow::MatvecPlan::kSymPartial
                        : use_cross ? skb_flow::MatvecPlan::kSymComplete
                                    : skb_flow::MatvecPlan::kPlain;
    // target lists of apply_matvec: r_all = [fibers | shell | bodies] (system.cpp:284-291),
    // r_fibbody = [fibers | bodies] (system.cpp:301-303), both restricted to this rank's pieces
    std::vector<double> r_win, r_fb;
    r_win.reserve((size_t)fl->n_win * 3);
    r_win.insert(r_win.end(), fl->h_r_fib.begin() + 3 * fl->fa, fl->h_r_fib.begin() + 3 * fl->fb);
    r_win.insert(r_win.end(), fl->h_r_shell.begin() + 3 * fl->sa, fl->h_r_shell.begin() + 3 * fl->sb);
    r_win.insert(r_win.end(), fl->h_r_body.begin() + 3 * fl->ba, fl->h_r_body.begin() + 3 * fl->bb);
    if (!use_cross)
        r_fb.insert(r_fb.end(), fl->h_r_fib.begin() + 3 * fl->fa, fl->h_r_fib.begin() + 3 * fl->fb);
    r_fb.insert(r_fb.end(), fl->h_r_body.begin() + 3 * fl->ba, fl->h_r_body.begin() + 3 * fl->bb);
    Evaluator &ef = fl->fib[1];
    std::vector<double> r_own; // the fiber evaluator's targets when they are not r_win
    if (sym_partial) {
        // fiber sources meet [ALL fiber nodes | own shell rows | own body rows]; with the cross kernel the periphery
        // rows are not targets of this evaluator
        r_own.reserve((size_t)(nf + n_sw + n_bw) * 3);
        r_own.insert(r_own.end(), fl->h_r_fib.begin(), fl->h_r_fib.end());
        if (!use_cross)
            r_own.insert(r_own.end(), fl->h_r_shell.begin() + 3 * fl->sa, fl->h_r_shell.begin() + 3 * fl->sb);
        r_own.insert(r_own.end(), fl->h_r_body.begin() + 3 * fl->ba, fl->h_r_body.begin() + 3 * fl->bb);
        ef.sym_mode = 1;
        ef.sym_part = fl->grp.rank();
        ef.sym_parts = fl->grp.size();
    } else {
        if (use_cross) { // [own fiber rows | own body rows]
            r_own.assign(fl->h_r_fib.begin() + 3 * fl->fa, fl->h_r_fib.begin() + 3 * fl->fb);
            r_own.insert(r_own.end(), fl->h_r_body.begin() + 3 * fl->ba, fl->h_r_body.begin() + 3 * fl->bb);
        }
        ef.sym_part = 0;
        ef.sym_parts = 1;
    }
    const std::vector<double> &r_ef = sym_partial || use_cross ? r_own : r_win;
    SKB_TRY(ef.set_targets(r_ef.data(), (long long)r_ef.size() / 3, false, fl->stream));
    SKB_TRY(fl->body[1].set_targets(r_win.data(), fl->n_win, false, fl->stream));
    SKB_TRY(fl->shell[1].set_targets(r_fb.data(), (long long)r_fb.size() / 3, false, fl->stream));
    CUDA_TRY(cudaStreamSynchronize(fl->stream));
    const bool all_fibers_lead = (fl->fa == 0 && fl->fb == nf) || sym_partial;
    if (fl->self_excl && fl->n_fib > 0) {
        if (!all_fibers_lead)
            return set_error(SKB_ERR_INVALID, "skb_flow_set_self_exclusion needs all fiber nodes as the leading matvec "
                                              "targets (no target window / ranges that cut the fiber rows)");
        std::vector<int32_t> ids((size_t)nf);
        for (int f = 0; f < fl->n_fibers; ++f)
            for (long long i = fl->h_fiber_off[(size_t)f]; i < fl->h_fiber_off[(size_t)f + 1]; ++i)
                ids[(size_t)i] = f;
        SKB_TRY(ef.set_exclusion_ids(ids.data(), nf, fl->stream));
        CUDA_TRY(cudaStreamSynchronize(fl->stream));
    } else {
        SKB_TRY(ef.set_exclusion_ids(nullptr, 0, fl->stream));
    }
    fl->mv_dirty = false;
    return SKB_OK;
}

// ---- matvec_core and its steps, on fl->cur -----------------------------------------------------------------------
// The pending dense product of apply_matvec_core goes out on the side stream, ordered after everything on fl->cur so far
// (its input is complete), and runs beside whatever fl->cur launches next.  The side stream has the highest priority:
// its one-warp CTAs (one per SM) are placed before the pair kernel's CTAs fill the SMs.
int skb::overlap_buffers(skb_flow *fl, long long n_rows) {
    skb_flow::Overlap &B = fl->bg;
    if (!B.stream) {
        int lo = 0, hi = 0;
        CUDA_TRY(cudaDeviceGetStreamPriorityRange(&lo, &hi));
        CUDA_TRY(cudaStreamCreateWithPriority(B.stream.out(), cudaStreamNonBlocking, hi));
        CUDA_TRY(cudaEventCreateWithFlags(B.fork.out(), cudaEventDisableTiming));
        CUDA_TRY(cudaEventCreateWithFlags(B.join.out(), cudaEventDisableTiming));
        // nothing may be loaded lazily later, while a group member on this device spins on a flag (the streamer itself
        // was loaded when the device was prepared, prepare_device)
        cudaFuncAttributes fa;
        CUDA_TRY(cudaFuncGetAttributes(&fa, add_out_kernel));
    }
    SKB_TRY(B.y.ensure((size_t)n_rows * 8 + 8));
    return SKB_OK;
}

// the complete x_shell on this device, input of the periphery's dense operator: the caller's vector without a group;
// with one, the gathered copy in the window half (epoch parity) of the group matvec in flight
static const double *full_x_shell(const skb_flow *fl, const double *d_xs) {
    return fl->grp.member() ? fl->grp.x_shell() : d_xs;
}

static int overlap_launch(skb_flow *fl, const double *d_xs) {
    skb_flow::Overlap &B = fl->bg;
    if (!B.dn || B.launched)
        return SKB_OK;
    CUDA_TRY(cudaEventRecord(B.fork, fl->cur));
    CUDA_TRY(cudaStreamWaitEvent(B.stream, B.fork, 0));
    SKB_TRY(skb_dense_apply_background_device(B.dn, SKB_DENSE_STRESSLET_PLUS_COMPLEMENTARY, full_x_shell(fl, d_xs),
                                              (double *)B.y.ptr, B.stream));
    CUDA_TRY(cudaEventRecord(B.join, B.stream));
    B.launched = true;
    fl->launches += 1;
    return SKB_OK;
}

// v = fc.flow(r_all, fw, eta)  (system.cpp:299) at the fiber evaluator's targets.  Symmetric producers: the symmetric
// kernel writes the fiber rows -- complete, or in a group this member's partial sums for ALL fiber rows into its
// window -- and the plain kernel the rest: [own periphery rows (not with the cross kernel) | own body rows]
static int fiber_rows(skb_flow *fl, StrengthMode mode, const double *ff, double eta, double *d_v) {
    const skb_flow::MatvecPlan &P = fl->plan;
    if (P.fib_rows == skb_flow::MatvecPlan::kPlain)
        return fibers_dev(fl, fl->fib[1], mode, ff, eta, 0, d_v, 0, fl->fa, fl->fb);
    const Group &G = fl->grp;
    const long long nf = fl->n_fib, n_fw = fl->fb - fl->fa, n_sw = fl->sb - fl->sa, n_bw = fl->bb - fl->ba;
    Evaluator &ef = fl->fib[1];
    SKB_TRY(fl->scratch_u.ensure((size_t)ef.n_trg * 24 + 8));
    EvalOpts o;
    o.d_u_sym = P.grouped ? G.u_part() : d_v;
    o.d_u_rem = d_v + 3 * (n_fw + (P.cross ? n_sw : 0));
    SKB_TRY(ef.eval(SKB_STOKESLET, mode, ff, 0.0, (double *)fl->scratch_u.ptr, 0, fl->cur, &fl->launches, nullptr,
                    1.0 / eta, o));
    fl->pairs += nf * nf / (P.grouped ? G.size() : 1) + nf * ((P.cross ? 0 : n_sw) + n_bw);
    if (ef.last_was_sym)
        return SKB_OK;
    if (P.grouped)
        return set_error(SKB_ERR_STATE, "group member %d: the symmetric kernel declined (memory for the reverse "
                                        "partials?); lower SKB_SYM_MAX_BYTES pressure or use fewer nodes per GPU",
                         G.rank());
    // the symmetric path declined (memory): everything landed contiguously in the scratch buffer
    CUDA_TRY(cudaMemcpyAsync(d_v, fl->scratch_u.ptr, (size_t)n_fw * 24, cudaMemcpyDeviceToDevice, fl->cur));
    if (n_bw > 0)
        CUDA_TRY(cudaMemcpyAsync(o.d_u_rem, (const double *)fl->scratch_u.ptr + 3 * n_fw, (size_t)n_bw * 24,
                                 cudaMemcpyDeviceToDevice, fl->cur));
    return SKB_OK;
}

// fiber <-> periphery pairs in one geometry pass (cross_kernels.cuh): stresslet sums of every periphery node (packed
// strengths s6) at the own fiber rows, Stokeslet sums of the own fibers at every periphery row.  Without a group both
// are complete: the fiber rows add onto the fiber-fiber sums, the periphery rows are written.  In a group the fiber rows
// are written (the fiber-fiber sums come with the pull), the Stokeslet sums are this member's partials in its window,
// and the own periphery rows start from zero until the members' partials are pulled in.
static int cross_rows(skb_flow *fl, const double *s6, double eta, double *d_v) {
    const bool grouped = fl->plan.grouped;
    const long long ns = fl->n_shell, n_fw = fl->fb - fl->fa, n_sw = fl->sb - fl->sa;
    const Evaluator &ef = fl->fib[1];
    const SourceSet &sf = ef.src[SKB_STOKESLET], &ss = fl->shell[1].src[SKB_STRESSLET];
    double *u_shell = grouped ? fl->grp.u_part_shell() : d_v + 3 * n_fw;
    SKB_TRY(cross_eval(fl->cross, ef.info, (const double *)sf.r.ptr, sf.f_cur, fl->fa, n_fw, (const double *)ss.r.ptr,
                       s6, ns, ss.n_pad, -3.0 / (8.0 * M_PI * eta), 1.0 / (8.0 * M_PI * eta), d_v, grouped ? 0 : 1,
                       u_shell, 0, fl->cur, &fl->launches));
    fl->pairs += 2 * n_fw * ns;
    if (grouped && n_sw > 0)
        CUDA_TRY(cudaMemsetAsync(d_v + 3 * n_fw, 0, (size_t)n_sw * 24, fl->cur));
    return SKB_OK;
}

// v_fibers, v_bodies += shell.flow(r_fibbody, x_shell, eta)  (system.cpp:304,313-315) through tmp.  The periphery
// evaluator's targets are [own fiber rows | own body rows], the body rows only when the cross kernel covers the fiber
// rows.  A group member's symmetric path has not written its fiber rows yet: they are set here (copied, or zeroed
// without periphery) and the pull adds the fiber-fiber sums.
static int periphery_rows(skb_flow *fl, StrengthMode mode, const double *sd, double eta, double *d_v) {
    const long long ns = fl->n_shell, n_fw = fl->fb - fl->fa, n_sw = fl->sb - fl->sa, n_bw = fl->bb - fl->ba;
    const long long n_fr = fl->plan.cross ? 0 : n_fw; // fiber rows among the periphery evaluator's targets
    const bool set_fib = fl->plan.fib_rows == skb_flow::MatvecPlan::kSymPartial;
    if (ns == 0 || n_fr + n_bw == 0) {
        if (set_fib && n_fr > 0)
            CUDA_TRY(cudaMemsetAsync(d_v, 0, (size_t)n_fr * 24, fl->cur));
        return SKB_OK;
    }
    SKB_TRY(fl->tmp.ensure((size_t)(n_fr + n_bw) * 24 + 8));
    double *d_tmp = (double *)fl->tmp.ptr;
    SKB_TRY(periphery_dev(fl, fl->shell[1], mode, sd, eta, d_tmp, 0));
    const int bs = 256;
    if (n_fr > 0 && set_fib) {
        CUDA_TRY(cudaMemcpyAsync(d_v, d_tmp, (size_t)n_fr * 24, cudaMemcpyDeviceToDevice, fl->cur));
    } else if (n_fr > 0) {
        add_inplace_kernel<<<(unsigned)((3 * n_fr + bs - 1) / bs), bs, 0, fl->cur>>>(d_v, d_tmp, 3 * n_fr);
        SKB_TRY(launched(&fl->launches));
    }
    if (n_bw > 0) {
        add_inplace_kernel<<<(unsigned)((3 * n_bw + bs - 1) / bs), bs, 0, fl->cur>>>(d_v + 3 * (n_fw + n_sw),
                                                                                  d_tmp + 3 * n_fr, 3 * n_bw);
        SKB_TRY(launched(&fl->launches));
    }
    return SKB_OK;
}

int skb::matvec_core(skb_flow *fl, const double *d_ff, const double *d_sd, const double *d_bd, const double *d_f,
                     const double *d_t, double eta, double *d_v) {
    const skb_flow::MatvecPlan &P = fl->plan;
    Group &G = fl->grp;
    const long long n_fw = fl->fb - fl->fa, n_sw = fl->sb - fl->sa;
    // strengths as the caller ships them (packed by the evaluations), or packed by the push into the group window
    StrengthMode fmode = kRaw, smode = kNormalDensity;
    const double *ff = d_ff, *sd = d_sd;
    if (P.grouped) {
        if (!fl->grp_open)
            SKB_TRY(G.begin());
        const Evaluator &ef = fl->fib[1];
        const SourceSet &sf = ef.src[SKB_STOKESLET];
        SKB_TRY(G.push(d_ff, sf.has_weights ? (const double *)sf.weights.ptr : nullptr, fl->fa, n_fw, d_sd,
                       fl->n_shell ? (const double *)fl->shell[1].src[SKB_STRESSLET].normals.ptr : nullptr,
                       fl->sa, n_sw, 2.0 * eta, ef.info.num_sms, fl->cur, &fl->launches));
        const bool ft = fl->ft_exchange && fl->n_bodies > 0; // d_f / d_t: this member's partial link forces
        if (ft)
            SKB_TRY(G.push_forces(d_f, d_t, fl->cur, &fl->launches));
        SKB_TRY(G.barrier(0, true, true, fl->cur, &fl->launches)); // every member's strengths have landed here
        if (ft) { // the bodies' link forces and torques: the members' partials in rank order (body_container.cpp:134)
            double *sum = (double *)fl->ft_sum.ptr;
            SKB_TRY(G.reduce_forces(sum, sum + 3 * fl->n_bodies, fl->cur, &fl->launches));
            d_f = sum;
            d_t = sum + 3 * fl->n_bodies;
        }
        fmode = smode = kPacked;
        ff = G.f_sl();
        sd = G.f_shell();
    } else if (fl->n_win == 0) {
        return SKB_OK;
    }
    SKB_TRY(overlap_launch(fl, d_sd)); // (x_shell is complete on this device from here on)
    SKB_TRY(fiber_rows(fl, fmode, ff, eta, d_v));
    // The self term subtracts from the fiber rows: without a group right after the fiber flow; a group member
    // subtracts it last, once the pull has completed its fiber rows (the plain-kernel member keeps that order too).
    if (!P.grouped)
        SKB_TRY(fiber_self_term(fl, fl->fib[1], eta, d_v, fl->fa, fl->fb));
    if (P.cross) {
        if (!P.grouped) { // periphery strengths 2 eta n (x) rho -> sym6 (periphery.cpp:68-71), once for both uses
            Evaluator &es = fl->shell[1];
            SKB_TRY(es.pack(SKB_STRESSLET, kNormalDensity, d_sd, 2.0 * eta, fl->cur, &fl->launches));
            smode = kPacked;
            sd = es.src[SKB_STRESSLET].f_cur;
        }
        SKB_TRY(cross_rows(fl, sd, eta, d_v));
    }
    const bool partial = P.fib_rows == skb_flow::MatvecPlan::kSymPartial;
    if (partial)
        SKB_TRY(G.barrier(1, true, false, fl->cur, &fl->launches)); // my partial sums are complete
    SKB_TRY(periphery_rows(fl, smode, sd, eta, d_v));
    // v_all += bc.flow(r_all, x_bodies, body_link_conditions, eta)     (system.cpp:316)
    SKB_TRY(bodies_dev(fl, fl->body[1], d_bd, d_f, d_t, eta, d_v, 1));
    if (partial) {
        SKB_TRY(G.barrier(1, false, true, fl->cur, &fl->launches));
        SKB_TRY(G.pull(Group::kFiberRows, fl->fa, n_fw, d_v, fl->cur, &fl->launches));
        if (P.cross) // own periphery rows += the members' Stokeslet partials
            SKB_TRY(G.pull(Group::kShellRows, fl->sa, n_sw, d_v + 3 * n_fw, fl->cur, &fl->launches));
    }
    if (P.grouped)
        SKB_TRY(fiber_self_term(fl, fl->fib[1], eta, d_v, fl->fa, fl->fb));
    return SKB_OK;
}

extern "C" {

int skb_flow_matvec(skb_flow *fl, const double *fib_forces, const double *shell_density, const double *body_densities,
                    const double *body_forces_torques, double eta, double *v_all) {
    if (!fl || !(eta > 0))
        return set_error(SKB_ERR_INVALID, "skb_flow_matvec: bad arguments");
    const long long nf = fl->n_fib, ns = fl->n_shell, nb = fl->n_body, n_all = nf + ns + nb;
    if ((nf > 0 && !fib_forces) || (ns > 0 && !shell_density) || (nb > 0 && !body_densities) ||
        (fl->n_bodies > 0 && !body_forces_torques) || (n_all > 0 && !v_all))
        return set_error(SKB_ERR_INVALID, "skb_flow_matvec: NULL input for a non-empty class");
    CUDA_TRY(cudaSetDevice(fl->dev));
    begin_stats(fl);
    if (n_all == 0)
        return SKB_OK;
    SKB_TRY(prepare_matvec_targets(fl));
    const long long n_win = fl->n_win;
    if (n_win == 0)
        return SKB_OK;
    std::vector<double> f, t;
    if (fl->n_bodies > 0)
        split_forces_torques(body_forces_torques, fl->n_bodies, f, t);
    Transfers xfer{{up(fib_forces, 3 * nf), up(shell_density, 3 * ns), up(body_densities, 3 * nb),
                    up(f.data(), f.size()), up(t.data(), t.size())},
                   {down(v_all, 3 * n_win)}};
    unsigned long long key = mix_key(fl->geom_version, (unsigned long long)fl->fa);
    key = mix_key(key, (unsigned long long)fl->n_win);
    key = mix_key(key, dbl_bits(eta));
    return replayable_call(fl, fl->g_matvec, 1, key, xfer, [&](const Transfers &io) {
        return matvec_core(fl, io.up[0].dev, io.up[1].dev, io.up[2].dev, io.up[3].dev, io.up[4].dev, eta,
                           io.down[0].dev);
    });
}

int skb_flow_matvec_device(skb_flow *fl, const double *d_fib_forces, const double *d_shell_density,
                           const double *d_body_densities, const double *d_body_forces, const double *d_body_torques,
                           double eta, double *d_v_window, void *stream) {
    if (!fl || !(eta > 0))
        return set_error(SKB_ERR_INVALID, "skb_flow_matvec_device: bad arguments");
    const long long nf = fl->n_fib, ns = fl->n_shell, nb = fl->n_body, n_all = nf + ns + nb;
    if ((nf > 0 && !d_fib_forces) || (ns > 0 && !d_shell_density) || (nb > 0 && !d_body_densities) ||
        (fl->n_bodies > 0 && (!d_body_forces || !d_body_torques)))
        return set_error(SKB_ERR_INVALID, "skb_flow_matvec_device: NULL input for a non-empty class");
    CUDA_TRY(cudaSetDevice(fl->dev));
    begin_stats(fl);
    if (n_all == 0)
        return SKB_OK;
    SKB_TRY(prepare_matvec_targets(fl));
    if (fl->n_win > 0 && !d_v_window)
        return set_error(SKB_ERR_INVALID, "skb_flow_matvec_device: NULL output");
    return device_frame(fl, stream, [&] {
        return matvec_core(fl, d_fib_forces, d_shell_density, d_body_densities, d_body_forces, d_body_torques, eta,
                           d_v_window);
    });
}

} // extern "C"

int skb::apply_matvec_core(skb_flow *fl, skb_dense *dn, const double *d_x, const double *d_xs, const double *d_bd,
                           const double *d_f, const double *d_t, const double *d_link, double eta, double *d_res_fib,
                           double *d_out_shell, double *d_v_bodies) {
    const long long n_fw = fl->fb - fl->fa, n_sw = fl->sb - fl->sa, n_bw = fl->bb - fl->ba;
    SKB_TRY(fl->fw.ensure((size_t)n_fw * 24 + 8));
    SKB_TRY(fl->vel.ensure((size_t)fl->n_win * 24 + 8));
    // res_shell's dense part, stresslet_plus_complementary_ * x_shell (system.cpp:319, periphery.cpp:38-47), depends on
    // x_shell only: it is handed to the background streamer, which matvec_core launches as soon as x_shell is complete
    // on this device (full_x_shell)
    skb_flow::Overlap &B = fl->bg;
    B.dn = nullptr;
    B.launched = false;
    const bool dense_rows = dn && n_sw > 0 && d_out_shell;
    if (dense_rows && B.enabled) {
        SKB_TRY(overlap_buffers(fl, 3 * n_sw));
        B.dn = dn;
    }
    // MatrixXd fw = fc.apply_fiber_force(x_fibers)                       system.cpp:298
    SKB_TRY(fl->ops.force(d_x, (double *)fl->fw.ptr, fl->cur, &fl->launches));
    // v_all of system.cpp:299-316 (own rows)
    SKB_TRY(matvec_core(fl, (const double *)fl->fw.ptr, d_xs, d_bd, d_f, d_t, eta, (double *)fl->vel.ptr));
    // res_fibers = fc.matvec(x_fibers, v_fibers, fiber_link_conditions)   system.cpp:318
    SKB_TRY(fl->ops.matvec(d_x, (const double *)fl->vel.ptr, d_link, d_res_fib, fl->cur, &fl->launches));
    const double *d_v_shell = (const double *)fl->vel.ptr + 3 * n_fw;
    if (n_sw > 0 && d_out_shell) {
        if (dense_rows && B.launched) {
            // res_shell = A x (background) + v_shell
            CUDA_TRY(cudaStreamWaitEvent(fl->cur, B.join, 0));
            add_out_kernel<<<(unsigned)((3 * n_sw + 255) / 256), 256, 0, fl->cur>>>(d_out_shell, (const double *)B.y.ptr,
                                                                                   d_v_shell, 3 * n_sw);
            SKB_TRY(launched(&fl->launches));
        } else if (dn) {
            // res_shell = shell.matvec(x_shell, v_shell) = stresslet_plus_complementary_ * x_shell + v_shell in one
            // kernel at the end of the stream (skb_flow_set_overlap(fl, 0))
            SKB_TRY(skb_dense_apply_device(dn, SKB_DENSE_STRESSLET_PLUS_COMPLEMENTARY, full_x_shell(fl, d_xs), d_v_shell,
                                           d_out_shell, fl->cur));
            fl->launches += 1;
        } else {
            CUDA_TRY(cudaMemcpyAsync(d_out_shell, d_v_shell, (size_t)n_sw * 24, cudaMemcpyDeviceToDevice, fl->cur));
        }
    }
    B.dn = nullptr;
    if (n_bw > 0 && d_v_bodies)
        CUDA_TRY(cudaMemcpyAsync(d_v_bodies, (const double *)fl->vel.ptr + 3 * (n_fw + n_sw), (size_t)n_bw * 24,
                                 cudaMemcpyDeviceToDevice, fl->cur));
    return SKB_OK;
}

// shared body of skb_flow_apply_matvec / skb_flow_apply_matvec_dense; dn != NULL: out_shell = res_shell
static int apply_matvec_impl(skb_flow *fl, skb_dense *dn, const double *x_fibers, const double *shell_density,
                             const double *body_densities, const double *body_forces_torques,
                             const double *fiber_link_conditions, double eta, double *res_fibers, double *v_shell,
                             double *v_bodies) {
    if (!fl || !(eta > 0))
        return set_error(SKB_ERR_INVALID, "skb_flow_apply_matvec: bad arguments");
    if (fl->n_fibers > 0) // no fibers: the empty operator set, uploaded or not
        SKB_TRY(fl->ops.ready("skb_flow_apply_matvec"));
    const long long nf = fl->n_fib, ns = fl->n_shell, nb = fl->n_body, n_all = nf + ns + nb;
    if ((nf > 0 && (!x_fibers || !res_fibers)) || (ns > 0 && (!shell_density || !v_shell)) ||
        (nb > 0 && (!body_densities || !v_bodies)) || (fl->n_bodies > 0 && !body_forces_torques))
        return set_error(SKB_ERR_INVALID, "skb_flow_apply_matvec: NULL argument for a non-empty class");
    CUDA_TRY(cudaSetDevice(fl->dev));
    begin_stats(fl);
    if (n_all == 0)
        return SKB_OK;
    SKB_TRY(prepare_matvec_targets(fl));
    if (fl->n_win != n_all || fl->grp.member())
        return set_error(SKB_ERR_INVALID, "skb_flow_apply_matvec needs the full target window (have %lld of %lld "
                                          "rows); group members use skb_flow_apply_matvec_device / skb_mflow_*",
                         fl->n_win, n_all);
    std::vector<double> f, t;
    if (fl->n_bodies > 0)
        split_forces_torques(body_forces_torques, fl->n_bodies, f, t);
    const bool link = nf && fiber_link_conditions;
    Transfers xfer{{up(x_fibers, 4 * nf), up(link ? fiber_link_conditions : nullptr, 7LL * fl->ops.n_fibers()),
                    up(shell_density, 3 * ns), up(body_densities, 3 * nb), up(f.data(), f.size()),
                    up(t.data(), t.size())},
                   {down(res_fibers, 4 * nf), down(v_shell, 3 * ns), down(v_bodies, 3 * nb)}};
    return host_call(fl, xfer, [&](const Transfers &io) {
        return apply_matvec_core(fl, dn, io.up[0].dev, io.up[2].dev, io.up[3].dev, io.up[4].dev, io.up[5].dev,
                                 link ? io.up[1].dev : nullptr, eta, io.down[0].dev, io.down[1].dev, io.down[2].dev);
    });
}

extern "C" {

int skb_flow_apply_matvec(skb_flow *fl, const double *x_fibers, const double *shell_density,
                          const double *body_densities, const double *body_forces_torques,
                          const double *fiber_link_conditions, double eta, double *res_fibers, double *v_shell,
                          double *v_bodies) {
    return apply_matvec_impl(fl, nullptr, x_fibers, shell_density, body_densities, body_forces_torques,
                             fiber_link_conditions, eta, res_fibers, v_shell, v_bodies);
}

int skb_flow_apply_matvec_dense(skb_flow *fl, skb_dense *dn, const double *x_fibers, const double *x_shell,
                                const double *body_densities, const double *body_forces_torques,
                                const double *fiber_link_conditions, double eta, double *res_fibers,
                                double *res_shell, double *v_bodies) {
    if (!fl || !dn)
        return set_error(SKB_ERR_INVALID, "skb_flow_apply_matvec_dense: NULL handle");
    SKB_TRY(dense_rows(fl, dn, "skb_flow_apply_matvec_dense", false));
    return apply_matvec_impl(fl, dn, x_fibers, x_shell, body_densities, body_forces_torques, fiber_link_conditions,
                             eta, res_fibers, res_shell, v_bodies);
}

int skb_flow_apply_matvec_device(skb_flow *fl, skb_dense *dn, const double *d_x_fibers, const double *d_x_shell,
                                 const double *d_body_densities, const double *d_body_forces,
                                 const double *d_body_torques, const double *d_fiber_link_conditions, double eta,
                                 double *d_res_fibers, double *d_out_shell, double *d_v_bodies, void *stream) {
    if (!fl || !(eta > 0))
        return set_error(SKB_ERR_INVALID, "skb_flow_apply_matvec_device: bad arguments");
    if (fl->n_fibers > 0)
        SKB_TRY(fl->ops.ready("skb_flow_apply_matvec_device"));
    CUDA_TRY(cudaSetDevice(fl->dev));
    begin_stats(fl);
    SKB_TRY(prepare_matvec_targets(fl));
    if (dn)
        SKB_TRY(dense_rows(fl, dn, "skb_flow_apply_matvec_device", false));
    const long long n_fw = fl->fb - fl->fa, n_sw = fl->sb - fl->sa, n_bw = fl->bb - fl->ba;
    if ((n_fw > 0 && (!d_x_fibers || !d_res_fibers)) || (n_sw > 0 && (!d_x_shell || !d_out_shell)) ||
        (fl->n_body > 0 && !d_body_densities) || (n_bw > 0 && !d_v_bodies) ||
        (fl->n_bodies > 0 && (!d_body_forces || !d_body_torques)))
        return set_error(SKB_ERR_INVALID, "skb_flow_apply_matvec_device: NULL argument for a non-empty class");
    if (!fl->grp.member() && fl->n_win == 0)
        return SKB_OK;
    if (!fl->grp.member() && fl->n_win != fl->n_fib + fl->n_shell + fl->n_body)
        return set_error(SKB_ERR_INVALID, "skb_flow_apply_matvec_device: a flow that owns only part of the rows must be a "
                                          "group member (skb_flow_group_init): the fiber forces of the other rows' "
                                          "fibers have to come from somewhere");
    return device_frame(fl, stream, [&] {
        return apply_matvec_core(fl, dn, d_x_fibers, d_x_shell, d_body_densities, d_body_forces, d_body_torques,
                                 d_fiber_link_conditions, eta, d_res_fibers, d_out_shell, d_v_bodies);
    });
}

} // extern "C"

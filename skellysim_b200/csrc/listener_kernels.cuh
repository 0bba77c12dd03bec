// listener_kernels.cuh -- the listener's kernels (skb_listener.cu): the frame of a step (the packing of
// trajectory_reader.cpp:238-246 and the bodies' [U; omega]), the body-interior replacement of
// System::velocity_at_targets (system.cpp:362-381) and the lockstep Cash-Karp 5(4) integration of many streamlines or
// vortex lines (streamline.cpp with boost.odeint's integrate_adaptive / controlled_runge_kutta).
//
// Every line (a seed and a direction) advances one try_step per attempt.  An attempt is six stages; each stage writes
// the stage points of the active lines into one compacted target array (slot j of the last compaction is line
// slots[j]), the flow evaluates them in one pass, and the next stage's kernel reads the velocities back by slot.
#pragma once
#include "skb_internal.hpp" // BodyItem
#include <cuda_runtime.h>

namespace skb {

constexpr int kLineThreads = 128;
constexpr int kStateThreads = 128;
constexpr int kCompactThreads = 1024;
constexpr int kLineMaxFails = 500;   // odeint's failed_step_checker
constexpr double kVortexEps = 1e-7;  // get_vorticity_at_point (streamline.cpp:16-35)
constexpr double kSingularSpeed = 1e3; // push_back_points_and_time: "Possible singularity detected"

// per body of the interior replacement: kind (0 none, 1 sphere, 2 ellipsoid), radii[3], centre[3], U[3], omega[3]
constexpr int kRigidStride = 13;

// the interior test of the body with rigid-table row p at x (kind 0: never inside); d = x - centre.  Every
// operation rounds on its own (no contraction), as the reference's separate products and sums do
__device__ __forceinline__ bool inside_body(const double *p, double x0, double x1, double x2, double &d0, double &d1,
                                            double &d2) {
    const int kind = (int)p[0];
    if (kind == 0)
        return false;
    d0 = __dsub_rn(x0, p[4]), d1 = __dsub_rn(x1, p[5]), d2 = __dsub_rn(x2, p[6]);
    if (kind == 1) {
        const double n2 = __dadd_rn(__dadd_rn(__dmul_rn(d0, d0), __dmul_rn(d1, d1)), __dmul_rn(d2, d2));
        return __dsqrt_rn(n2) < p[1];
    }
    const double q0 = __ddiv_rn(__ddiv_rn(__dmul_rn(d0, d0), p[1]), p[1]);
    const double q1 = __ddiv_rn(__ddiv_rn(__dmul_rn(d1, d1), p[2]), p[2]);
    const double q2 = __ddiv_rn(__ddiv_rn(__dmul_rn(d2, d2), p[3]), p[3]);
    return __dadd_rn(__dadd_rn(q0, q1), q2) < 1.0;
}

// points inside a body take the body's rigid motion U + omega x dx; bodies in order, the last match wins
__global__ void interior_replace_kernel(const double *__restrict__ trg, long long n_trg,
                                        const double *__restrict__ rigid, int n_bodies, double *__restrict__ vel) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_trg)
        return;
    const double x0 = trg[3 * i], x1 = trg[3 * i + 1], x2 = trg[3 * i + 2];
    for (int b = 0; b < n_bodies; ++b) {
        const double *p = rigid + (size_t)b * kRigidStride;
        double d0, d1, d2;
        if (inside_body(p, x0, x1, x2, d0, d1, d2)) {
            const double w0 = p[10], w1 = p[11], w2 = p[12];
            vel[3 * i] = __dadd_rn(p[7], __dsub_rn(__dmul_rn(w1, d2), __dmul_rn(w2, d1)));
            vel[3 * i + 1] = __dadd_rn(p[8], __dsub_rn(__dmul_rn(w2, d0), __dmul_rn(w0, d2)));
            vel[3 * i + 2] = __dadd_rn(p[9], __dsub_rn(__dmul_rn(w0, d1), __dmul_rn(w1, d0)));
        }
    }
}

// The gradient's last pass: g (10 per target, gradient_dev) splits into grad (9 per target) and the pressure, which
// gradient_dev leaves over eta.  Inside a body (the test and order of interior_replace_kernel) the gradient is the
// rigid motion's, d u_i / d x_j = eps_ikj omega_k, and the pressure NaN: a rigid body has no fluid pressure
__global__ void gradient_finish_kernel(const double *__restrict__ trg, long long n_trg, const double *__restrict__ rigid,
                                       int n_bodies, double eta, const double *__restrict__ g, double *__restrict__ grad,
                                       double *__restrict__ pressure) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_trg)
        return;
    double o[10];
    for (int k = 0; k < 10; ++k)
        o[k] = g[10 * i + k];
    o[9] *= eta;
    const double x0 = trg[3 * i], x1 = trg[3 * i + 1], x2 = trg[3 * i + 2];
    for (int b = 0; b < n_bodies; ++b) {
        const double *p = rigid + (size_t)b * kRigidStride;
        double d0, d1, d2;
        if (inside_body(p, x0, x1, x2, d0, d1, d2)) {
            const double w0 = p[10], w1 = p[11], w2 = p[12];
            const double r[10] = {0.0, -w2, w1, w2, 0.0, -w0, -w1, w0, 0.0, __longlong_as_double(0x7ff8000000000000LL)};
            for (int k = 0; k < 10; ++k)
                o[k] = r[k];
        }
    }
    for (int k = 0; k < 9; ++k)
        grad[9 * i + k] = o[k];
    pressure[i] = o[9];
}

// The frame of skb_flow_set_listener_state, one launch of n_fibers + n_bodies CTAs.  CTA f < n_fibers packs fiber f's
// solution block [x; y; z; T] (4n, the layout fiber_gemv_kernel<1> and fiber_link_kernel read) from the installed
// positions (3 per node) and the tension (1 per node), as trajectory_reader.cpp:238-246 fills sol_fibers from x_ and
// tension_.  CTA n_fibers + b writes body b's [U; omega], the last six entries of its block of x_bodies
// (SphericalBody::step, body_spherical.cpp:16-17), into its row of the rigid table.  Copies only: no rounding
__global__ void __launch_bounds__(kStateThreads)
    listener_state_kernel(const long long *__restrict__ fib_off, int n_fibers, const double *__restrict__ r_fib,
                          const double *__restrict__ tension, double *__restrict__ x_fib,
                          const BodyItem *__restrict__ bodies, const double *__restrict__ x_bodies,
                          double *__restrict__ rigid) {
    const int blk = blockIdx.x;
    if (blk < n_fibers) {
        const long long o = fib_off[blk];
        const int n = (int)(fib_off[blk + 1] - o);
        double *x = x_fib + 4 * o;
        for (int i = threadIdx.x; i < n; i += kStateThreads) {
            const double *r = r_fib + 3 * (o + i);
            x[i] = r[0];
            x[n + i] = r[1];
            x[2 * n + i] = r[2];
            x[3 * n + i] = tension[o + i];
        }
        return;
    }
    const int b = blk - n_fibers;
    if (threadIdx.x < 6) {
        const BodyItem it = bodies[b];
        rigid[(size_t)b * kRigidStride + 7 + threadIdx.x] = x_bodies[it.sol_off + 3LL * it.n_nodes + threadIdx.x];
    }
}

// ---- the lines -------------------------------------------------------------------------------------------------
// line l = 2 i + d: seed i, direction d (0 back to -t_final, 1 forward to +t_final)
enum : int { kLineActive = -1, kLineReached = 0, kLineSingular = 1, kLineFailed = 2, kLineCapped = 3 };

struct LineState {
    double *x;     // 3 per line: the state
    double *t, *dt;
    double *k;     // 18 per line: k1..k6 of the attempt in flight
    int *status;   // kLineActive or the exit
    int *count;    // points written
    int *fails;    // consecutive failed tries of the current step
    int *pending;  // the state was accepted (or is the seed) and is not observed yet
    double *out_x, *out_t, *out_val; // max_points per line: 3, 1, 3 doubles per point
    const int *slots;                // slot -> line of the last compaction
};

struct LineParams {
    double t_final, abs_err, rel_err;
    int max_points, vortex;
};

// points per line and stage: a streamline's one; a vortex line's six x +- eps e_j and x itself (the observer's
// velocity at stage 1).  Every stage of an attempt evaluates the same number of points, so that a stage point equal
// to x (dt below x's rounding) gets exactly k1, as the reference's repeated evaluations at one point do
__host__ __device__ __forceinline__ int line_points(int vortex) { return vortex ? 7 : 1; }

// Cash-Karp 5(4) (runge_kutta_cash_karp54): a_ij, the 5th-order weights b and b - b* of the error estimate
__device__ __forceinline__ double ck_a(int s, int j) { // stage s (2..6), j < s - 1
    switch (s) {
    case 2: return 1.0 / 5.0;
    case 3: return j == 0 ? 3.0 / 40.0 : 9.0 / 40.0;
    case 4: return j == 0 ? 3.0 / 10.0 : j == 1 ? -9.0 / 10.0 : 6.0 / 5.0;
    case 5: return j == 0 ? -11.0 / 54.0 : j == 1 ? 5.0 / 2.0 : j == 2 ? -70.0 / 27.0 : 35.0 / 27.0;
    default:
        return j == 0 ? 1631.0 / 55296.0 : j == 1 ? 175.0 / 512.0 : j == 2 ? 575.0 / 13824.0
             : j == 3 ? 44275.0 / 110592.0 : 253.0 / 4096.0;
    }
}
__device__ __forceinline__ double ck_b(int j) {
    const double b[6] = {37.0 / 378.0, 0.0, 250.0 / 621.0, 125.0 / 594.0, 0.0, 512.0 / 1771.0};
    return b[j];
}
__device__ __forceinline__ double ck_db(int j) {
    const double db[6] = {37.0 / 378.0 - 2825.0 / 27648.0, 0.0, 250.0 / 621.0 - 18575.0 / 48384.0, 125.0 / 594.0 - 13525.0 / 55296.0,
                          0.0 - 277.0 / 14336.0, 512.0 / 1771.0 - 1.0 / 4.0};
    return db[j];
}

// odeint's less_with_sign(t1, t2, dt)
__device__ __forceinline__ bool less_with_sign(double t1, double t2, double dt) {
    return dt > 0 ? t2 - t1 > 2.220446049250313e-16 : t1 - t2 > 2.220446049250313e-16;
}

// the derivative of slot j from the velocities of a stage with `np` points per slot: the velocity, or the vorticity
// of the six central differences exactly as get_vorticity_at_point combines them
__device__ __forceinline__ void line_derivative(const double *__restrict__ vel, long long j, int np, int vortex,
                                                double k[3]) {
    const double *v = vel + 3 * (size_t)j * np;
    if (!vortex) {
        k[0] = v[0];
        k[1] = v[1];
        k[2] = v[2];
        return;
    }
    // v(c, p) = v[3 p + c]
    k[0] = __ddiv_rn(__dmul_rn(0.5, __dsub_rn(__dsub_rn(v[3 * 2 + 2], v[3 * 3 + 2]), __dsub_rn(v[3 * 4 + 1], v[3 * 5 + 1]))),
                     kVortexEps);
    k[1] = __ddiv_rn(__dmul_rn(0.5, __dsub_rn(__dsub_rn(v[3 * 4 + 0], v[3 * 5 + 0]), __dsub_rn(v[3 * 0 + 2], v[3 * 1 + 2]))),
                     kVortexEps);
    k[2] = __ddiv_rn(__dmul_rn(0.5, __dsub_rn(__dsub_rn(v[3 * 0 + 1], v[3 * 1 + 1]), __dsub_rn(v[3 * 2 + 0], v[3 * 3 + 0]))),
                     kVortexEps);
}

// the seeds: line 2 i + d starts at x0[i], t = 0, dt = +-dt_init; without back integration the back lines are done
// with no points
__global__ void line_init_kernel(LineState s, const double *__restrict__ x0, int n_lines, double dt_init, int back) {
    const int l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= 2 * n_lines)
        return;
    const int i = l >> 1, d = l & 1;
    for (int c = 0; c < 3; ++c)
        s.x[3 * l + c] = x0[3 * i + c];
    s.t[l] = 0.0;
    s.dt[l] = d ? dt_init : -dt_init;
    s.status[l] = (d == 0 && !back) ? kLineReached : kLineActive;
    s.count[l] = 0;
    s.fails[l] = 0;
    s.pending[l] = 1;
}

// slots <- the active lines in line order, *n_act <- their count: one block, a scan per chunk of the lines
__global__ void __launch_bounds__(kCompactThreads) line_compact_kernel(const int *__restrict__ status, int n,
                                                                       int *__restrict__ slots, int *__restrict__ n_act) {
    __shared__ int warp_sum[kCompactThreads / 32];
    __shared__ int base;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0)
        base = 0;
    __syncthreads();
    for (int c0 = 0; c0 < n; c0 += kCompactThreads) {
        const int l = c0 + tid;
        const int a = l < n && status[l] == kLineActive;
        int incl = a; // inclusive scan in the warp
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o)
                incl += y;
        }
        if (lane == 31)
            warp_sum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            int w = warp_sum[lane];
            for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o)
                    w += y;
            }
            warp_sum[lane] = w; // inclusive over the warps
        }
        __syncthreads();
        const int before = base + (warp ? warp_sum[warp - 1] : 0) + incl - a;
        if (a)
            slots[before] = l;
        __syncthreads();
        if (tid == 0)
            base += warp_sum[kCompactThreads / 32 - 1];
        __syncthreads();
    }
    if (tid == 0)
        *n_act = base;
}

// Stage s (1..6) of the attempt of slot j < n_slots.  From stage 2 on it first stores k_{s-1} from the previous
// stage's velocities (vel_prev, line_points(vortex) per slot).  At stage 2 a line whose state is not observed
// yet is observed (integrate_adaptive's obs(x, t), with the velocity at x from stage 1): the point is appended, and the
// line ends at |v| > 1e3, at +-t_final or at its max_points-th point; otherwise dt is cut to land on +-t_final and the
// step's failure count starts at 0.  Then the stage points x + dt sum_j a_sj k_j go to trg (a line that ended here
// writes x, which nothing reads).
__global__ void line_stage_kernel(LineState s, LineParams p, int stage, int n_slots, const double *__restrict__ vel_prev,
                                  double *__restrict__ trg) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_slots)
        return;
    const int l = s.slots[j];
    double x[3] = {s.x[3 * l], s.x[3 * l + 1], s.x[3 * l + 2]};
    double dt = s.dt[l];
    bool live = s.status[l] == kLineActive;
    if (stage >= 2 && live) {
        const int np = line_points(p.vortex);
        double k[3];
        line_derivative(vel_prev, j, np, p.vortex, k);
        for (int c = 0; c < 3; ++c)
            s.k[18 * l + 3 * (stage - 2) + c] = k[c];
        if (stage == 2 && s.pending[l]) {
            s.pending[l] = 0;
            const double *v = p.vortex ? vel_prev + 3 * ((size_t)j * np + 6) : vel_prev + 3 * (size_t)j;
            const int n = s.count[l];
            const size_t o = (size_t)l * p.max_points + n;
            const double t = s.t[l];
            for (int c = 0; c < 3; ++c) {
                s.out_x[3 * o + c] = x[c];
                s.out_val[3 * o + c] = k[c];
            }
            s.out_t[o] = t;
            s.count[l] = n + 1;
            const double T = (l & 1) ? p.t_final : -p.t_final;
            const double speed = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
            int st = kLineActive;
            if (speed > kSingularSpeed)
                st = kLineSingular;
            else if (!less_with_sign(t, T, dt))
                st = kLineReached;
            else if (n + 1 >= p.max_points)
                st = kLineCapped;
            if (st != kLineActive) {
                s.status[l] = st;
                live = false;
            } else {
                if (less_with_sign(T, t + dt, dt)) {
                    dt = T - t;
                    s.dt[l] = dt;
                }
                s.fails[l] = 0;
            }
        }
    }
    if (live && stage >= 2) {
        // x + (dt a_s1) k1 + (dt a_s2) k2 + ..., each product and sum rounded on its own as odeint's scale_sum
        double acc[3] = {x[0], x[1], x[2]};
        for (int q = 0; q < stage - 1; ++q) {
            const double c = __dmul_rn(dt, ck_a(stage, q));
            for (int e = 0; e < 3; ++e)
                acc[e] = __dadd_rn(acc[e], __dmul_rn(c, s.k[18 * l + 3 * q + e]));
        }
        x[0] = acc[0];
        x[1] = acc[1];
        x[2] = acc[2];
    }
    double *o = trg + 3 * (size_t)j * line_points(p.vortex);
    if (!p.vortex) {
        o[0] = x[0];
        o[1] = x[1];
        o[2] = x[2];
        return;
    }
    for (int q = 0; q < 6; ++q) { // x_plus_eps.col(q): +eps, -eps along axis q / 2
        for (int e = 0; e < 3; ++e)
            o[3 * q + e] = x[e];
        o[3 * q + q / 2] = (q & 1) ? x[q / 2] - kVortexEps : x[q / 2] + kVortexEps;
    }
    for (int e = 0; e < 3; ++e)
        o[18 + e] = x[e];
}

// After stage 6: k6 from its velocities, the new state and the error estimate; controlled_runge_kutta::try_step's
// accept (t += dt, dt grown by the default step adjuster when err < 0.5, the state replaced and awaiting its
// observation) or reject (dt shrunk, the state kept; the 500th consecutive failure ends the line)
__global__ void line_control_kernel(LineState s, LineParams p, int n_slots, const double *__restrict__ vel) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_slots)
        return;
    const int l = s.slots[j];
    if (s.status[l] != kLineActive)
        return;
    double *k = s.k + 18 * (size_t)l;
    line_derivative(vel, j, line_points(p.vortex), p.vortex, k + 15);
    const double dt = s.dt[l];
    double x_new[3], err = 0.0;
    for (int c = 0; c < 3; ++c) {
        const double x = s.x[3 * l + c];
        double xn = x, xe = 0.0;
        for (int q = 0; q < 6; ++q) { // uncontracted, as the stage points: an error estimate of exactly 0 stays 0
            xn = __dadd_rn(xn, __dmul_rn(__dmul_rn(dt, ck_b(q)), k[3 * q + c]));
            xe = __dadd_rn(xe, __dmul_rn(__dmul_rn(dt, ck_db(q)), k[3 * q + c]));
        }
        x_new[c] = xn;
        // default_error_checker: |xerr| / (eps_abs + eps_rel (|x| + |dt| |dxdt|)); the maximum ignores NaN as
        // std::max(err, e) does
        const double e = __ddiv_rn(fabs(xe), __dadd_rn(p.abs_err, __dmul_rn(p.rel_err, __dadd_rn(fabs(x),
                                                                                         __dmul_rn(fabs(dt), fabs(k[c]))))));
        if (err < e)
            err = e;
    }
    if (err > 1.0) { // default_step_adjuster::decrease_step, error order 4
        const double f = 0.9 * pow(err, -1.0 / 3.0);
        s.dt[l] = dt * (f < 0.2 ? 0.2 : f);
        const int fails = s.fails[l] + 1;
        s.fails[l] = fails;
        if (fails >= kLineMaxFails)
            s.status[l] = kLineFailed;
        return;
    }
    s.t[l] += dt;
    double dt_new = dt;
    if (err < 0.5) { // increase_step, stepper order 5
        const double e = 1.0 / 3125.0 < err ? err : 1.0 / 3125.0;
        dt_new = dt * (0.9 * pow(e, -1.0 / 5.0));
    }
    s.dt[l] = dt_new;
    for (int c = 0; c < 3; ++c)
        s.x[3 * l + c] = x_new[c];
    s.pending[l] = 1;
}

} // namespace skb

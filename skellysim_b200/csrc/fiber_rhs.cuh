// fiber_rhs.cuh -- the fiber block of the right-hand side of one timestep formed on the device
// (skb_flow_build_fiber_rhs): RHS_ of every fiber as it stands after FiberFiniteDifference::update_RHS
// (fiber_finite_difference.cpp:198-274) and the RHS half of apply_bc_rectangular (:358-361 and the B_RHS lines of every
// boundary-condition branch, :377-383, 399-404, 422-423, 432-433, 455-463, 481-486, 502-504).
//
//   fiber_rhs_kernel  One CTA per fiber.  Positions, velocities and forces are staged in shared memory; xs_ and xss_
//       are formed by update_derivatives (fiber_build.cuh, K = 2), then v D_1 and f_tot D_1 with D_1 scaled by
//       length_, the raw 4n vector of update_RHS, rows [0, 4n-14) = P_downsample_bc * raw over each row's non-zero
//       column range (as the assembly does for A_), and the 14 boundary entries.
//
// f_tot = f_external + force_scale_ xs_ (System::prep_state_for_solver, system.cpp:416-451; the motor force of
// generate_constant_force, fcfd.cpp:160-169) feeds update_RHS; the boundary entries see f_external alone (system.cpp:453).
#pragma once
#include "fiber_build.cuh"

namespace skb {

constexpr int kRhsThreads = 128; // fiber_rhs_kernel

__host__ __device__ inline size_t rhs_smem_bytes(int n) { return (size_t)28 * n * sizeof(double); }

struct RhsArgs {
    const FiberItem *items;
    const FiberParamsDev *params;
    const double2 *growth; // per fiber: (v_growth_, force_scale_)
    const double *class_mats;
    const int2 *row_range;
    const double *r_fib;   // 3 x N_f, all fibers
    const double *length;  // length_ of every fiber of the container
    const double *v, *f;   // 3 x own nodes: flow at the fiber nodes, f_external; either may be NULL
    int motor;             // force_scale_ given: f_tot = f_external + force_scale_ xs_
    double dt, eta;
    double *rhs;           // 4 per own node
};

__global__ void __launch_bounds__(kRhsThreads) fiber_rhs_kernel(const RhsArgs a) {
    extern __shared__ double fr_smem[];
    const FiberItem it = a.items[blockIdx.x];
    const FiberParamsDev prm = a.params[blockIdx.x];
    const double2 gr = a.growth[blockIdx.x];
    const int n = it.n, m = 4 * n, bc = m - 14;
    double *xv = fr_smem;                  // [n x 3] positions
    double *vv = xv + 3 * n;               // [n x 3] flow (zero when NULL)
    double *fe = vv + 3 * n;               // [n x 3] f_external (zero when NULL)
    double *ft = fe + 3 * n;               // [n x 3] f_tot
    double *d1 = ft + 3 * n, *d2 = d1 + 3 * n; // xs_, xss_
    double *vD = d2 + 3 * n, *fD = vD + 3 * n; // v D_1, f_tot D_1
    double *raw = fD + 3 * n;              // [4n] update_RHS's RHS_
    const double *D1 = a.class_mats + it.cls; // pre-transposed: row i of D_k is D_k_0[i*n, i*n+n)
    const double *P = D1 + (size_t)n * n;
    const double *D2 = P + (size_t)bc * m;
    const bool has_v = a.v != nullptr, has_f = a.f != nullptr, has_ft = has_f || a.motor;

    for (int e = threadIdx.x; e < 3 * n; e += blockDim.x) {
        xv[e] = a.r_fib[3 * it.node + e];
        vv[e] = has_v ? a.v[3 * it.own_node + e] : 0.0;
        fe[e] = has_f ? a.f[3 * it.own_node + e] : 0.0;
    }
    __syncthreads();
    update_derivatives<2>(xv, D1, D2, n, 2.0 / prm.length_prev, d1);
    for (int e = threadIdx.x; e < 3 * n; e += blockDim.x) // (d1[e] was formed by this thread)
        ft[e] = a.motor ? fe[e] + gr.y * d1[e] : fe[e];
    __syncthreads();

    // update_RHS takes D_1 with length_ (ffd.cpp:201): (v D_1)_i = sum_j v_j D_1_0(j, i) 2 / length_
    const double L = a.length[it.fiber];
    const double s1 = 2.0 / L;
    for (int e = threadIdx.x; e < 3 * n; e += blockDim.x) {
        const int i = e / 3, c = e - 3 * i;
        double sv = 0.0, sf = 0.0;
        for (int j = 0; j < n; ++j) {
            const double dij = D1[i * n + j];
            sv = fma(dij, vv[3 * j + c], sv);
            sf = fma(dij, ft[3 * j + c], sf);
        }
        vD[e] = s1 * sv;
        fD[e] = s1 * sf;
    }
    __syncthreads();

    // update_constants (fiber_finite_difference.hpp:140-144)
    const double eps = prm.radius / L;
    const double c0 = -log(M_E * (eps * eps)) / (8.0 * M_PI * a.eta), c1 = 2.0 / (8.0 * M_PI * a.eta);
    // the raw RHS_ of update_RHS (ffd.cpp:211-273); s_dot = (1 + alpha) v_growth_ / 2, alpha = LinSpaced(n, -1, 1)
    for (int R = threadIdx.x; R < m; R += blockDim.x) {
        const int ra = R / n, i = R - ra * n;
        const double *xs = d1 + 3 * i, *xss = d2 + 3 * i, *f = ft + 3 * i, *v = vv + 3 * i;
        double r;
        if (ra < 3) {
            const double alpha = i == n - 1 ? 1.0 : -1.0 + i * (2.0 / (n - 1));
            const double s_dot = (1.0 + alpha) * (0.5 * gr.x);
            r = xv[3 * i + ra] / a.dt + s_dot * xs[ra];
            if (has_v)
                r += v[ra];
            if (has_ft) { // c_0 (I + xs xs^T) f + c_1 (I - xs xs^T) f
                const double xf = (xs[0] * f[0] + xs[1] * f[1]) + xs[2] * f[2];
                r += (c0 + c1) * f[ra] + ((c0 - c1) * xs[ra]) * xf;
            }
        } else {
            r = -prm.penalty_param;
            if (has_v)
                r += (xs[0] * vD[3 * i] + xs[1] * vD[3 * i + 1]) + xs[2] * vD[3 * i + 2];
            if (has_ft) {
                r += (2.0 * c0) * ((xs[0] * fD[3 * i] + xs[1] * fD[3 * i + 1]) + xs[2] * fD[3 * i + 2]);
                r += (c0 - c1) * ((xss[0] * f[0] + xss[1] * f[1]) + xss[2] * f[2]);
            }
        }
        raw[R] = r;
    }
    __syncthreads();

    // rows [0, 4n-14): P_downsample_bc * raw over the non-zero columns of each row of P                  (ffd.cpp:359)
    double *out = a.rhs + 4 * it.own_node;
    const int2 *rg = a.row_range + it.rng;
    for (int r = threadIdx.x; r < bc; r += blockDim.x) {
        const int2 cr = rg[r];
        double acc = 0.0;
        for (int c = cr.x; c < cr.y; ++c)
            acc = fma(P[r + (size_t)c * bc], raw[c], acc);
        out[r] = acc;
    }
    // the 14 entries of B_RHS: the minus end from node 0, the plus end from node n - 1, f_external only      (:360-504)
    if (threadIdx.x < 14) {
        const int t = threadIdx.x, end = t < 7 ? 0 : n - 1;
        const bool vel = t < 7 ? prm.minus_clamped : prm.plus_hinged;
        const double *x = xv + 3 * end, *xs = d1 + 3 * end, *f = fe + 3 * end, *v = vv + 3 * end;
        const int k = t < 7 ? t : t - 7; // 0-2 first condition, 3 its scalar row, 4-6 second condition
        double b = 0.0;
        if (k < 3) { // Velocity: x_ / dt; Force: f_external
            b = vel ? x[k] / a.dt : f[k];
        } else if (k == 3) {
            if (vel) { // -xs . v - 2 c_0 xs . f_external
                if (has_v)
                    b -= (xs[0] * v[0] + xs[1] * v[1]) + xs[2] * v[2];
                if (has_f)
                    b -= 2.0 * c0 * ((xs[0] * f[0] + xs[1] * f[1]) + xs[2] * f[2]);
            } else { // f_external . xs
                b = (f[0] * xs[0] + f[1] * xs[1]) + f[2] * xs[2];
            }
        } else if (t < 7 && vel) { // minus AngularVelocity: xs_ / dt; the Torque rows stay 0
            b = xs[k - 4] / a.dt;
        }
        out[bc + t] = b;
    }
}

} // namespace skb

// periphery_kernels.cuh -- the fiber-periphery repulsion, the periphery binding and the collision test of
// SphericalPeriphery / EllipsoidalPeriphery (periphery.cpp:94-97, 126-162, 204-263; fiber_finite_difference.cpp:74-91;
// fcfd.cpp:39-54; body_spherical.cpp:304-307) in one pass over the fiber positions (skb_periphery.cu).
#pragma once
#include "../../include/skelly_b200_flow.h" // SKB_PERIPHERY_*
#include <cuda_runtime.h>

namespace skb {

constexpr int kPeriThreads = 128;

// the shape as the kernel reads it (skb_periphery_shape)
struct PeriShape {
    int kind; // SKB_PERIPHERY_SPHERE or SKB_PERIPHERY_ELLIPSOID
    int binding;
    double a, b, c, f_0, l_0, start, end, threshold;
};

// per-fiber flags of periphery_kernel; the extra last entry holds kPeriCollided when two bodies or a body and the
// periphery collide
enum : int { kPeriHinged = 1, kPeriCollided = 2, kPeriNonFinite = 4 };

// the point of the ellipsoid (semi-axes shrunk by t) in the direction of x, with the reference's 1e-12 guards
// (periphery.cpp:207-214, 242-250)
__device__ __forceinline__ void peri_cortex(const PeriShape &s, const double x[3], double t, double rc[3]) {
    const double rs[3] = {x[0] / s.a, x[1] / s.b, x[2] / s.c};
    const double rs_mag = sqrt(rs[0] * rs[0] + rs[1] * rs[1] + rs[2] * rs[2]);
    const double phi = atan2(rs[1], rs[0] + 1e-12);
    const double theta = acos(rs[2] / (1e-12 + rs_mag));
    const double st = sin(theta);
    rc[0] = (s.a - t) * st * cos(phi);
    rc[1] = (s.b - t) * st * sin(phi);
    rc[2] = (s.c - t) * cos(theta);
}

// Periphery::check_collision of one point at threshold t: on or beyond the (shrunk) surface
__device__ __forceinline__ bool peri_outside(const PeriShape &s, const double x[3], double t) {
    const double r2 = x[0] * x[0] + x[1] * x[1] + x[2] * x[2];
    if (s.kind == SKB_PERIPHERY_SPHERE) {
        const double R = s.a - t;
        return r2 >= R * R;
    }
    double rc[3];
    peri_cortex(s, x, t, rc);
    return r2 >= rc[0] * rc[0] + rc[1] * rc[1] + rc[2] * rc[2];
}

// fiber_interaction of one node: f_0 dr / |dr| exp(-(R - |x|) / l_0) strictly inside the surface, else 0.  A node at
// the centre of a sphere divides 0 by 0, as the reference does (NaN)
__device__ __forceinline__ void peri_force(const PeriShape &s, const double x[3], double f[3]) {
    const double r_mag = sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
    double R, surf[3];
    if (s.kind == SKB_PERIPHERY_SPHERE) {
        R = s.a;
        for (int k = 0; k < 3; ++k)
            surf[k] = x[k] / r_mag * R;
    } else {
        peri_cortex(s, x, 0.0, surf);
        R = sqrt(surf[0] * surf[0] + surf[1] * surf[1] + surf[2] * surf[2]);
    }
    f[0] = f[1] = f[2] = 0.0;
    if (!(r_mag < R))
        return;
    const double dr[3] = {x[0] - surf[0], x[1] - surf[1], x[2] - surf[2]};
    const double d = sqrt(dr[0] * dr[0] + dr[1] * dr[1] + dr[2] * dr[2]);
    const double e = exp(-(R - r_mag) / s.l_0);
    for (int k = 0; k < 3; ++k)
        f[k] = s.f_0 * dr[k] / d * e;
}

// One block per fiber of [f0, f0 + gridDim.x - 1), the last block for the bodies.  Fiber f (node i at r_fib[3 i]):
//   force (not NULL): the repulsion of its nodes, 3 per node from node off[f0] on; node 0 is skipped (0) when
//     force_skip0[f] (minus_clamped_, periphery.cpp:148, 240);
//   flags[f - f0]: kPeriHinged = update_boundary_conditions' plus hinge (the binding window at the polar angle of its
//     last node and a node within the binding threshold of the surface), kPeriCollided = a node on or beyond the
//     surface (node 0 skipped when collide_skip0[f], is_minus_clamped()), kPeriNonFinite = a non-finite force.
// flags[gridDim.x - 1]: kPeriCollided when spherical bodies (radius > 0) overlap, or one reaches a sphere's surface.
// Each node's values depend on its position alone and the flags are block-level ORs: no launch-configuration effect
__global__ void __launch_bounds__(kPeriThreads)
    periphery_kernel(const PeriShape s, const double *__restrict__ r_fib, const long long *__restrict__ off, int f0,
                     const int *__restrict__ force_skip0, const int *__restrict__ collide_skip0,
                     double *__restrict__ force, const double *__restrict__ centers,
                     const double *__restrict__ radius, int n_bodies, int *__restrict__ flags) {
    const int nf = (int)gridDim.x - 1;
    if ((int)blockIdx.x == nf) { // the bodies: against each other (i < j) and against a sphere
        bool hit = false;
        const long long n_pairs = (long long)n_bodies * n_bodies;
        for (long long p = threadIdx.x; p < n_pairs; p += blockDim.x) {
            const int i = (int)(p / n_bodies), j = (int)(p % n_bodies);
            const double *ci = centers + 3 * i, ri = radius[i];
            if (ri <= 0.0)
                continue;
            if (i == j) {
                if (s.kind == SKB_PERIPHERY_SPHERE)
                    hit |= sqrt(ci[0] * ci[0] + ci[1] * ci[1] + ci[2] * ci[2]) + ri > s.a;
                continue;
            }
            const double rj = radius[j];
            if (j < i || rj <= 0.0)
                continue;
            const double *cj = centers + 3 * j;
            const double d[3] = {ci[0] - cj[0], ci[1] - cj[1], ci[2] - cj[2]};
            const double rr = ri + rj;
            hit |= d[0] * d[0] + d[1] * d[1] + d[2] * d[2] < rr * rr;
        }
        hit = __syncthreads_or(hit);
        if (threadIdx.x == 0)
            flags[nf] = hit ? kPeriCollided : 0;
        return;
    }
    const int f = f0 + (int)blockIdx.x;
    const long long n0 = off[f], n = off[f + 1] - n0, base = off[f0];
    const int fskip = force_skip0[f] ? 1 : 0, cskip = collide_skip0[f] ? 1 : 0;
    bool near = false, collided = false, bad = false;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
        const double *p = r_fib + 3 * (n0 + i);
        const double x[3] = {p[0], p[1], p[2]};
        near |= s.binding && peri_outside(s, x, s.threshold);
        collided |= i >= cskip && peri_outside(s, x, 0.0);
        if (force) {
            double fv[3] = {0.0, 0.0, 0.0};
            if (i >= fskip)
                peri_force(s, x, fv);
            bad |= !isfinite(fv[0]) || !isfinite(fv[1]) || !isfinite(fv[2]);
            double *o = force + 3 * (n0 + i - base);
            o[0] = fv[0];
            o[1] = fv[1];
            o[2] = fv[2];
        }
    }
    near = __syncthreads_or(near);
    collided = __syncthreads_or(collided);
    bad = __syncthreads_or(bad);
    if (threadIdx.x == 0) {
        // acos(x_last.normalized()[2]); Eigen's normalized() of a zero vector is the zero vector (angle pi/2)
        const double *q = r_fib + 3 * (n0 + n - 1);
        const double z2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2];
        const double angle = acos(z2 > 0.0 ? q[2] / sqrt(z2) : 0.0);
        const bool hinged = near && angle >= s.start && angle <= s.end;
        flags[blockIdx.x] = (hinged ? kPeriHinged : 0) | (collided ? kPeriCollided : 0) | (bad ? kPeriNonFinite : 0);
    }
}

// out = in + add (in == NULL: out = add), n doubles; out may be in
__global__ void periphery_add_kernel(const double *in, const double *__restrict__ add, double *out, long long n) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        out[i] = in ? in[i] + add[i] : add[i];
}

} // namespace skb

// aux_kernels.cuh -- small O(N) device kernels of the flow() layer (SkellySim fiber / periphery / body flows).
#pragma once
#include <cuda_runtime.h>

namespace skb {

// Per-fiber self-interaction, subtracted from the all-pairs velocity at the fiber's own nodes:
//   vel[off+i] -= sum_j G(x_i - x_j) wf_j,   G = regularised Oseen tensor / (8 pi eta)
// == `vel_flat -= fib.stokeslet_ * wf_flat` (fiber_container_finite_difference.cpp:203-210) with
// fib.stokeslet_ = kernels::oseen_tensor_direct(x_, x_, eta) (fiber_finite_difference.cpp:56,
// kernels.cpp:146-195: zero for r == 0, regularised by reg for 0 < r <= eps).  One CTA per fiber, one thread
// per node (n_nodes <= 128, fiber_finite_difference.cpp:522); the 3n x 3n matrix is never formed.
// `wf` are the trapezoid-weighted forces, i.e. the packed Stokeslet strengths.
__global__ void fiber_self_subtract_kernel(const double *__restrict__ r_fib, const double *__restrict__ wf,
                                           const long long *__restrict__ fiber_offset, double inv_8pi_eta,
                                           double reg2, double eps, double *__restrict__ vel, long long node_begin,
                                           long long node_end) {
    // only fiber nodes in [node_begin, node_end) are targets of this launch (target window of a rank);
    // vel is indexed window-locally: row (node - node_begin)
    extern __shared__ double sh[]; // [n*3 positions][n*3 strengths]
    const long long off = fiber_offset[blockIdx.x];
    const int n = (int)(fiber_offset[blockIdx.x + 1] - off);
    if (off + n <= node_begin || off >= node_end)
        return;
    double *xs = sh, *fs = sh + 3 * n;
    for (int i = threadIdx.x; i < 3 * n; i += blockDim.x) {
        xs[i] = r_fib[3 * off + i];
        fs[i] = wf[3 * off + i];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        if (off + i < node_begin || off + i >= node_end)
            continue;
        const double x = xs[3 * i], y = xs[3 * i + 1], z = xs[3 * i + 2];
        double a0 = 0, a1 = 0, a2 = 0;
        for (int j = 0; j < n; ++j) {
            const double dx = xs[3 * j] - x, dy = xs[3 * j + 1] - y, dz = xs[3 * j + 2] - z; // src - trg, kernels.cpp:161
            const double dr2 = dx * dx + dy * dy + dz * dz;
            if (dr2 == 0.0)
                continue;
            const double dr = sqrt(dr2);
            double fr, gr;
            if (dr > eps) {
                fr = inv_8pi_eta / dr;
                gr = inv_8pi_eta / (dr * dr * dr);
            } else {
                const double di = 1.0 / sqrt(dr * dr + reg2);
                fr = inv_8pi_eta * di;
                gr = inv_8pi_eta * di * di * di;
            }
            const double d0 = fs[3 * j], d1 = fs[3 * j + 1], d2 = fs[3 * j + 2];
            const double dot = gr * (dx * d0 + dy * d1 + dz * d2);
            a0 += fr * d0 + dx * dot;
            a1 += fr * d1 + dy * dot;
            a2 += fr * d2 + dz * dot;
        }
        const long long row = off + i - node_begin;
        vel[3 * row + 0] -= a0;
        vel[3 * row + 1] -= a1;
        vel[3 * row + 2] -= a2;
    }
}

// kernels::rotlet (kernels.cpp:206-242): u_t += 1/(8 pi eta) sum_s (L_s x d)/|d|^3, d = trg - src, regularised for
// |d|^2 < eps^2.  Sources are the few body centres, so one thread per target walks them all.
__global__ void rotlet_add_kernel(const double *__restrict__ r_src, const double *__restrict__ torque, int n_src,
                                  const double *__restrict__ r_trg, long long n_trg, double inv_8pi_eta, double reg2,
                                  double eps2, double *__restrict__ u) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_trg)
        return;
    const double x = r_trg[3 * t], y = r_trg[3 * t + 1], z = r_trg[3 * t + 2];
    double a0 = 0, a1 = 0, a2 = 0;
    for (int s = 0; s < n_src; ++s) {
        const double dx = x - r_src[3 * s], dy = y - r_src[3 * s + 1], dz = z - r_src[3 * s + 2];
        const double dr2 = dx * dx + dy * dy + dz * dz;
        const double dr = dr2 < eps2 ? sqrt(reg2 + dr2) : sqrt(dr2);
        const double fr = 1.0 / (dr * dr * dr);
        const double l0 = torque[3 * s], l1 = torque[3 * s + 1], l2 = torque[3 * s + 2];
        a0 += fr * (dz * l1 - dy * l2);
        a1 += fr * (dx * l2 - dz * l0);
        a2 += fr * (dy * l0 - dx * l1);
    }
    u[3 * t + 0] += inv_8pi_eta * a0;
    u[3 * t + 1] += inv_8pi_eta * a1;
    u[3 * t + 2] += inv_8pi_eta * a2;
}

// kernels::oseen_tensor_contract_direct (kernels.cpp:85-131) for a handful of point forces, accumulated into u:
// regularised for 0 < r <= eps, r == 0 skipped (point_source.cpp:42).  One thread per target.
__global__ void oseen_contract_add_kernel(const double *__restrict__ r_src, const double *__restrict__ density,
                                          int n_src, const double *__restrict__ r_trg, long long n_trg,
                                          double inv_8pi_eta, double reg2, double eps, double *__restrict__ u) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_trg)
        return;
    const double x = r_trg[3 * t], y = r_trg[3 * t + 1], z = r_trg[3 * t + 2];
    double a0 = 0, a1 = 0, a2 = 0;
    for (int s = 0; s < n_src; ++s) {
        const double dx = r_src[3 * s] - x, dy = r_src[3 * s + 1] - y, dz = r_src[3 * s + 2] - z; // kernels.cpp:100-102
        const double dr2 = dx * dx + dy * dy + dz * dz;
        const double dr = sqrt(dr2);
        if (dr == 0.0)
            continue;
        double fr, gr;
        if (dr > eps) {
            fr = inv_8pi_eta / dr;
            gr = inv_8pi_eta / (dr * dr * dr);
        } else {
            const double di = 1.0 / sqrt(dr * dr + reg2);
            fr = inv_8pi_eta * di;
            gr = inv_8pi_eta * di * di * di;
        }
        const double d0 = density[3 * s], d1 = density[3 * s + 1], d2 = density[3 * s + 2];
        const double dot = gr * (dx * d0 + dy * d1 + dz * d2);
        a0 += fr * d0 + dx * dot;
        a1 += fr * d1 + dy * dot;
        a2 += fr * d2 + dz * dot;
    }
    u[3 * t + 0] += a0;
    u[3 * t + 1] += a1;
    u[3 * t + 2] += a2;
}

// ---- the gradients of the velocities above (skb_flow_listener_gradient): 10 per target, d u_i / d x_j at 3 i + j and
// the pressure over eta at 9.  r = trg - src; the regularised branch is the velocity kernel's at that distance, with
// d|r|_reg / d r_j = r_j / |r|_reg in both branches; a coincident pair adds exactly 0 (the reference's r == 0 rule).
// rotlet_add_kernel's u = c (L x r) / D^3:  G_ij = c (eps_iaj L_a / D^3 - 3 (L x r)_i r_j / D^5), no pressure
__global__ void rotlet_grad_add_kernel(const double *__restrict__ r_src, const double *__restrict__ torque, int n_src,
                                       const double *__restrict__ r_trg, long long n_trg, double inv_8pi_eta,
                                       double reg2, double eps2, double *__restrict__ g) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_trg)
        return;
    const double x = r_trg[3 * t], y = r_trg[3 * t + 1], z = r_trg[3 * t + 2];
    double a[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int s = 0; s < n_src; ++s) {
        const double d[3] = {x - r_src[3 * s], y - r_src[3 * s + 1], z - r_src[3 * s + 2]};
        const double dr2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
        if (dr2 == 0.0)
            continue;
        const double dr = dr2 < eps2 ? sqrt(reg2 + dr2) : sqrt(dr2);
        const double fr = 1.0 / (dr * dr * dr), hr = 3.0 * fr / (dr * dr);
        const double l0 = torque[3 * s], l1 = torque[3 * s + 1], l2 = torque[3 * s + 2];
        const double m[3] = {d[2] * l1 - d[1] * l2, d[0] * l2 - d[2] * l0, d[1] * l0 - d[0] * l1}; // L x r
        const double e[9] = {0, -l2, l1, l2, 0, -l0, -l1, l0, 0};                               // eps_iaj L_a
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j)
                a[3 * i + j] += fr * e[3 * i + j] - hr * m[i] * d[j];
    }
    for (int k = 0; k < 9; ++k)
        g[10 * t + k] += inv_8pi_eta * a[k];
}

// oseen_contract_add_kernel's u = c (f / D + r (r.f) / D^3):
//   G_ij = c ((delta_ij (r.f) + r_i f_j - f_i r_j) / D^3 - 3 r_i r_j (r.f) / D^5),  p / eta = 2 c (r.f) / D^3
// with r = trg - src (the velocity kernel's src - trg is even; the pressure is odd)
__global__ void oseen_grad_add_kernel(const double *__restrict__ r_src, const double *__restrict__ density, int n_src,
                                      const double *__restrict__ r_trg, long long n_trg, double inv_8pi_eta,
                                      double reg2, double eps, double *__restrict__ g) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_trg)
        return;
    const double x = r_trg[3 * t], y = r_trg[3 * t + 1], z = r_trg[3 * t + 2];
    double a[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int s = 0; s < n_src; ++s) {
        const double d[3] = {x - r_src[3 * s], y - r_src[3 * s + 1], z - r_src[3 * s + 2]};
        const double dr = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
        if (dr == 0.0)
            continue;
        const double D = dr > eps ? dr : sqrt(dr * dr + reg2);
        const double gr = 1.0 / (D * D * D), hr = 3.0 * gr / (D * D);
        const double f[3] = {density[3 * s], density[3 * s + 1], density[3 * s + 2]};
        const double rf = d[0] * f[0] + d[1] * f[1] + d[2] * f[2];
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j)
                a[3 * i + j] += gr * ((i == j ? rf : 0.0) + d[i] * f[j] - f[i] * d[j]) - hr * rf * d[i] * d[j];
        a[9] += 2.0 * gr * rf;
    }
    for (int k = 0; k < 10; ++k)
        g[10 * t + k] += inv_8pi_eta * a[k];
}

// background_add_kernel's u_j = uniform_j + scale_j r[c_j]:  d u_j / d x_{c_j} += scale_j
__global__ void background_grad_add_kernel(long long n_trg, int c0, int c1, int c2, double s0, double s1, double s2,
                                           double *__restrict__ g) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_trg)
        return;
    g[10 * t + 0 + c0] += s0;
    g[10 * t + 3 + c1] += s1;
    g[10 * t + 6 + c2] += s2;
}

// BackgroundSource::flow (background_source.cpp:15-24): u_j += uniform_j + r[components_j] * scale_j
__global__ void background_add_kernel(const double *__restrict__ r_trg, long long n_trg, int c0, int c1, int c2,
                                      double s0, double s1, double s2, double u0, double u1, double u2,
                                      double *__restrict__ u) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_trg)
        return;
    u[3 * t + 0] += u0 + r_trg[3 * t + c0] * s0;
    u[3 * t + 1] += u1 + r_trg[3 * t + c1] * s1;
    u[3 * t + 2] += u2 + r_trg[3 * t + c2] * s2;
}

// dst[i] += src[i]
__global__ void add_inplace_kernel(double *__restrict__ dst, const double *__restrict__ src, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n)
        dst[i] += src[i];
}

// out[i] = a[i] + b[i]
__global__ void add_out_kernel(double *__restrict__ out, const double *__restrict__ a, const double *__restrict__ b,
                               long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n)
        out[i] = a[i] + b[i];
}

// per-node trapezoid weights 0.5 * L * weights_0 (fiber_container_finite_difference.cpp:186,
// fiber_finite_difference.cpp:545-548): weights_0 = 2/(n-1), halved at both ends
__global__ void fiber_weights_kernel(const long long *__restrict__ fiber_offset, const double *__restrict__ length,
                                     int n_fibers, double *__restrict__ w) {
    const int f = blockIdx.x;
    if (f >= n_fibers)
        return;
    const long long off = fiber_offset[f];
    const int n = (int)(fiber_offset[f + 1] - off);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        double w0 = 2.0;
        if (i == 0 || i == n - 1)
            w0 = 1.0;
        w[off + i] = 0.5 * length[f] * (w0 / (double)(n - 1));
    }
}

} // namespace skb

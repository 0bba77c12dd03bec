// body_ops.cuh -- the body block of System::apply_matvec and the fiber-body links, device resident (BodyOps,
// skb_body.cu).  Citations are `file:line` in the SkellySim tree.
//
//   fiber_link_kernel    BodyContainer::calculate_link_conditions (body_container.cpp:196-264) per fiber: the 7 link
//                        conditions fc.matvec takes (zeros for a free fiber, :177) and the fiber's force / torque on its
//                        body.  One warp per fiber; xss_0 / xsss_0 as a fixed-order warp reduction over the nodes.
//   body_sum_kernel      the bodies' link forces / torques (:240-241): per body the contributions of its bound fibers
//                        added in container order (no atomics: the sums are bitwise reproducible), and the body
//                        densities gathered out of x_bodies into the 3 x N_b layout of the body flow (:286-289).
//   body_matvec_kernel   SphericalBody::matvec (body_spherical.cpp:39-63; EllipsoidalBody::matvec is the same code) per
//                        body: the node rows and the 6 rows -K^T lambda + U with a fixed-order reduction tree.
//                        <true>: the rows a group member of skb_mflow owns (BodyOps, skb_internal.hpp).
//   system_rhs_rows_kernel  the shell and body rows of System::prep_state_for_solver's RHS: -v, and six zeros per body.
//   body_place_kernel    a rigid body's operators at rotation R from those of its body frame (skb_flow_place_bodies,
//                        DESIGN.md §3.6): A_^-1 = Q A_0^-1 Q^T, Q = blockdiag(R, ..., R), one 3 x 3 tile at a time,
//                        and per node E_i = R E_i,0 R^T, E_i = [ex_i ey_i ez_i].
// K_ is never stored: K U = u + w x (x_i - c) and K^T lambda = [sum lambda_i ; sum (x_i - c) x lambda_i]
// (update_K_matrix, body_spherical.cpp:74-86).
#pragma once
#include "skb_internal.hpp" // BodyItem
#include <cuda_runtime.h>

namespace skb {

struct LinkFiber {         // one fiber of the flow, in container order
    double s[3];           // nucleation site - body centre (body_container.cpp:209); unused for a free fiber
    double rigidity;       // bending_rigidity_
    long long node_off;    // first node of the fiber (x_fibers at 4 node_off, xs_ at 3 node_off)
    long long d2_off;      // element offset of its class's D_2_0 in the class table; D_3_0 follows (n x n each)
    int n_nodes;
    int body;              // -1: free
};

constexpr int kLinkWarps = 4;    // fibers per CTA of fiber_link_kernel
constexpr int kBodyThreads = 256; // threads per body of body_sum_kernel / body_matvec_kernel

__device__ __forceinline__ void cross3(const double *a, const double *b, double *c) {
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}

// link [7 per fiber], contrib [6 per bound fiber's index]: F_body, L_body.  x_fib: per fiber [x; y; z; T] of 4n;
// xs: the resident tangents xs_ (3 per node); length: length_ per fiber; class_mats: FiberOps' class table
__global__ void __launch_bounds__(32 * kLinkWarps)
    fiber_link_kernel(const LinkFiber *__restrict__ fibers, int n_fibers, const BodyItem *__restrict__ bodies,
                      const double *__restrict__ class_mats, const double *__restrict__ xs,
                      const double *__restrict__ length, const double *__restrict__ x_fib,
                      const double *__restrict__ x_bodies, double *__restrict__ link, double *__restrict__ contrib) {
    const int lane = threadIdx.x & 31;
    const int f = blockIdx.x * kLinkWarps + (int)(threadIdx.x >> 5);
    if (f >= n_fibers)
        return;
    const LinkFiber lf = fibers[f];
    if (lf.body < 0) { // body_container.cpp:177,203-204
        if (lane < 7)
            link[7LL * f + lane] = 0.0;
        return;
    }
    const int n = lf.n_nodes;
    const double *x = x_fib + 4 * lf.node_off;
    const double *D2 = class_mats + lf.d2_off, *D3 = D2 + (long long)n * n;
    // column 0 of x_new * D_k_0 (:218-221): sum_j x[:, j] D_k_0(j, 0)
    double a2[3] = {0.0, 0.0, 0.0}, a3[3] = {0.0, 0.0, 0.0};
    for (int j = lane; j < n; j += 32) {
        const double d2 = D2[j], d3 = D3[j];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const double xk = x[k * n + j];
            a2[k] = fma(xk, d2, a2[k]);
            a3[k] = fma(xk, d3, a3[k]);
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            a2[k] += __shfl_xor_sync(0xffffffffu, a2[k], o);
            a3[k] += __shfl_xor_sync(0xffffffffu, a3[k], o);
        }
    if (lane != 0)
        return;
    const double q = 2.0 / length[f];
    const double q2 = q * q, q3 = q2 * q;
    double xss[3], xsss[3], xs0[3], U[3], w[3];
    const BodyItem b = bodies[lf.body];
    const double *Uw = x_bodies + b.sol_off + 3LL * b.n_nodes; // body_velocities (:184-194)
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        xss[k] = q2 * a2[k];
        xsss[k] = q3 * a3[k];
        xs0[k] = xs[3 * lf.node_off + k];
        U[k] = Uw[k];
        w[k] = Uw[3 + k];
    }
    const double T0 = x[3 * n];
    const double E = lf.rigidity;
    const double *s = lf.s;
    double s_xsss[3], s_xs[3], xs_xss[3], w_s[3], xs_s[3], sn[3], sn_w[3];
    cross3(s, xsss, s_xsss);
    cross3(s, xs0, s_xs);
    cross3(xs0, xss, xs_xss);
    cross3(w, s, w_s);
    cross3(xs0, s, xs_s);
    const double inv_norm = 1.0 / sqrt(s[0] * s[0] + s[1] * s[1] + s[2] * s[2]);
#pragma unroll
    for (int k = 0; k < 3; ++k)
        sn[k] = s[k] * inv_norm;
    cross3(sn, w, sn_w);
    double *lk = link + 7LL * f, *ct = contrib + 6LL * f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        ct[k] = -E * xsss[k] + xs0[k] * T0;                             // F_body  :226
        ct[3 + k] = -E * s_xsss[k] + s_xs[k] * T0 + E * xs_xss[k];      // L_body  :231-237
        lk[k] = -U[k] - w_s[k];                                         // v_fiber :249
        lk[4 + k] = sn_w[k];                                            // w_fiber :256
    }
    lk[3] = -(xs0[0] * U[0] + xs0[1] * U[1] + xs0[2] * U[2]) +
            (xs_s[0] * w[0] + xs_s[1] * w[1] + xs_s[2] * w[2]); // tension_condition :252
}

// one CTA per body.  csr_begin[b]..csr_begin[b+1]: its bound fibers in container order in csr_fib (csr_begin NULL: no
// fiber is bound, the sums are zero)
__global__ void __launch_bounds__(kBodyThreads)
    body_sum_kernel(const BodyItem *__restrict__ bodies, const int *__restrict__ csr_begin,
                    const int *__restrict__ csr_fib, const double *__restrict__ contrib,
                    const double *__restrict__ x_bodies, double *__restrict__ dens, double *__restrict__ force,
                    double *__restrict__ torque) {
    const int b = blockIdx.x;
    const BodyItem it = bodies[b];
    if (threadIdx.x < 6) {
        const int k = threadIdx.x;
        double acc = 0.0;
        if (csr_begin)
            for (int i = csr_begin[b]; i < csr_begin[b + 1]; ++i)
                acc += contrib[6LL * csr_fib[i] + k];
        (k < 3 ? force : torque)[3 * b + (k % 3)] = acc;
    }
    const double *src = x_bodies + it.sol_off;
    double *dst = dens + 3 * it.node_off;
    for (int i = threadIdx.x; i < 3 * it.n_nodes; i += kBodyThreads)
        dst[i] = src[i];
}

// res (x_bodies layout) of every body.  r: body node positions (3 per node), centers (3 per body), w: node_weights_,
// ex / ey / ez: the singularity-subtraction vectors (3 per node), v: v_bodies (3 per node).
// kWindow (a group member, BodyOps): bodies b_first + blockIdx.x; only the node rows of nodes in [lo, hi) and the six
// rows of a body whose first node is in [lo, hi) are written, v holds the nodes [lo, hi) only.  K^T lambda still sums
// over all of the body's nodes (x_bodies and the geometry are complete), in the same order as without the window.
template <bool kWindow>
__global__ void __launch_bounds__(kBodyThreads)
    body_matvec_kernel(const BodyItem *__restrict__ bodies, const double *__restrict__ r,
                       const double *__restrict__ centers, const double *__restrict__ wgt,
                       const double *__restrict__ ex, const double *__restrict__ ey, const double *__restrict__ ez,
                       const double *__restrict__ x_bodies, const double *__restrict__ v, double *__restrict__ res,
                       int b_first, long long lo, long long hi) {
    __shared__ double red[6][kBodyThreads];
    const int b = kWindow ? b_first + (int)blockIdx.x : (int)blockIdx.x;
    const BodyItem it = bodies[b];
    const int n = it.n_nodes;
    const double *x = x_bodies + it.sol_off;
    double *out = res + it.sol_off;
    const double u[3] = {x[3 * n], x[3 * n + 1], x[3 * n + 2]}, om[3] = {x[3 * n + 3], x[3 * n + 4], x[3 * n + 5]};
    const double c[3] = {centers[3 * b], centers[3 * b + 1], centers[3 * b + 2]};
    double acc[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int i = threadIdx.x; i < n; i += kBodyThreads) {
        const long long g = it.node_off + i;
        const double d[3] = {x[3 * i], x[3 * i + 1], x[3 * i + 2]};
        const double rr[3] = {r[3 * g] - c[0], r[3 * g + 1] - c[1], r[3 * g + 2] - c[2]};
        const double dx = d[0] / wgt[g], dy = d[1] / wgt[g], dz = d[2] / wgt[g];
        double om_r[3], r_d[3];
        cross3(om, rr, om_r);
        cross3(rr, d, r_d);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            if (!kWindow || (g >= lo && g < hi)) {
                const double cxyz = dx * ex[3 * g + k] + dy * ey[3 * g + k] + dz * ez[3 * g + k];
                out[3 * i + k] = -cxyz - (u[k] + om_r[k]) + v[3 * (g - (kWindow ? lo : 0)) + k]; // :60
            }
            acc[k] += d[k];
            acc[3 + k] += r_d[k];
        }
    }
#pragma unroll
    for (int k = 0; k < 6; ++k)
        red[k][threadIdx.x] = acc[k];
    __syncthreads();
    for (int h = kBodyThreads / 2; h > 0; h >>= 1) {
        if ((int)threadIdx.x < h)
#pragma unroll
            for (int k = 0; k < 6; ++k)
                red[k][threadIdx.x] += red[k][threadIdx.x + h];
        __syncthreads();
    }
    if (threadIdx.x < 6 && (!kWindow || (it.node_off >= lo && it.node_off < hi)))
        out[3 * n + threadIdx.x] = -red[threadIdx.x][0] + x[3 * n + threadIdx.x]; // res_com = -K^T lambda + U  :61
}

// The shell and body rows of System::prep_state_for_solver's RHS (system.cpp:448,455): Periphery::update_RHS
// (periphery.cpp:86) rhs_shell = -v_shell, and per body update_RHS (body_spherical.cpp:134-138) [-v of its nodes ; six
// zeros].  CTAs [0, n_body_ctas) take the bodies b_first + blockIdx.x: the node rows of nodes in [lo, hi) (v holds the
// nodes [lo, hi)) and the six rows of a body whose first node is in [lo, hi), of rhs_bodies in the x_bodies layout --
// the rows a group member owns, or every row with lo = 0, hi = N_b.  The other CTAs negate the n_shell3 shell entries.
__global__ void __launch_bounds__(kBodyThreads)
    system_rhs_rows_kernel(const BodyItem *__restrict__ bodies, int b_first, int n_body_ctas, long long lo,
                           long long hi, const double *__restrict__ v, double *__restrict__ rhs_bodies,
                           const double *__restrict__ v_shell, long long n_shell3, double *__restrict__ rhs_shell) {
    if ((int)blockIdx.x >= n_body_ctas) {
        const long long stride = (long long)(gridDim.x - n_body_ctas) * kBodyThreads;
        for (long long i = (long long)(blockIdx.x - n_body_ctas) * kBodyThreads + threadIdx.x; i < n_shell3; i += stride)
            rhs_shell[i] = -v_shell[i];
        return;
    }
    const BodyItem it = bodies[b_first + (int)blockIdx.x];
    double *out = rhs_bodies + it.sol_off;
    const long long a = max(lo, it.node_off), e = min(hi, it.node_off + it.n_nodes);
    for (long long k = 3 * a + threadIdx.x; k < 3 * e; k += kBodyThreads)
        out[k - 3 * it.node_off] = -v[k - 3 * lo];
    if (threadIdx.x < 6 && it.node_off >= lo && it.node_off < hi)
        out[3 * it.n_nodes + threadIdx.x] = 0.0;
}

// ---- placement of a rigid body (body_place_kernel) ----
// Every entry of A_ and of ex_ / ey_ / ez_ depends on the nodes only through differences of positions, their norms and
// dot products with the normals, and K_ through x_i - c: placing the body at (c, R) maps A_0 to Q A_0 Q^T, so its
// inverse to Q A_0^-1 Q^T, and E_i,0 to R E_i,0 R^T.  (3n + 6 is a multiple of 3: the [U; w] rows and columns form two
// more tiles that R rotates like the node tiles.)
struct PlaceBody {       // one body whose inverse is kept
    long long inv_off;   // element offset of its (3n+6)^2 column-major inverse in the kept inverses
    int m;               // 3n + 6
    int body;            // index of its rotation
    int cta0;            // first CTA of its column tiles (one CTA per 3 columns)
    int pad;
};

constexpr int kPlaceThreads = 256;
constexpr int kPlaceRows = 3 * kPlaceThreads; // rows of a column tile staged per pass

// Y = R X R^T of one 3 x 3 tile, x[q][p] = X(p, q): Z = X R^T, then Y = R Z, each entry a three-term FMA chain
__device__ __forceinline__ void rotate_tile(const double (&R)[9], const double (&x)[3][3], double (&y)[3][3]) {
    double z[3][3];
#pragma unroll
    for (int p = 0; p < 3; ++p)
#pragma unroll
        for (int b = 0; b < 3; ++b)
            z[b][p] = fma(x[2][p], R[3 * b + 2], fma(x[1][p], R[3 * b + 1], x[0][p] * R[3 * b]));
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b)
            y[b][a] = fma(R[3 * a + 2], z[b][2], fma(R[3 * a + 1], z[b][1], R[3 * a] * z[b][0]));
}

// CTAs [0, n_inv_ctas): one column tile (3 consecutive columns, contiguous in the column-major inverse) of a kept
// inverse each, streamed through shared memory in passes of kPlaceRows rows -- coalesced loads of X0, each thread
// rotates one 3 x 3 tile in place, coalesced stores of X.  CTAs n_inv_ctas + b: body b's nodes, E_i = R E_i,0 R^T.
// R: 9 per body, row-major.
__global__ void __launch_bounds__(kPlaceThreads)
    body_place_kernel(const PlaceBody *__restrict__ place, int n_place, int n_inv_ctas, const BodyItem *__restrict__ bodies,
                      const double *__restrict__ R, const double *__restrict__ X0, double *__restrict__ X,
                      const double *__restrict__ ex0, const double *__restrict__ ey0, const double *__restrict__ ez0,
                      double *__restrict__ ex, double *__restrict__ ey, double *__restrict__ ez) {
    __shared__ double tile[3][kPlaceRows];
    const int t = threadIdx.x;
    if ((int)blockIdx.x >= n_inv_ctas) {
        const int b = (int)blockIdx.x - n_inv_ctas;
        const BodyItem it = bodies[b];
        double Rb[9];
#pragma unroll
        for (int k = 0; k < 9; ++k)
            Rb[k] = R[9 * b + k];
        for (int i = t; i < it.n_nodes; i += kPlaceThreads) {
            const long long g = 3 * (it.node_off + i);
            double e[3][3], y[3][3];
#pragma unroll
            for (int p = 0; p < 3; ++p) {
                e[0][p] = ex0[g + p];
                e[1][p] = ey0[g + p];
                e[2][p] = ez0[g + p];
            }
            rotate_tile(Rb, e, y);
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                ex[g + a] = y[0][a];
                ey[g + a] = y[1][a];
                ez[g + a] = y[2][a];
            }
        }
        return;
    }
    int lo = 0, hi = n_place - 1; // the last body whose cta0 <= blockIdx.x
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (place[mid].cta0 <= (int)blockIdx.x)
            lo = mid;
        else
            hi = mid - 1;
    }
    const PlaceBody pb = place[lo];
    const int m = pb.m;
    const long long col = 3LL * ((int)blockIdx.x - pb.cta0);
    const double *src = X0 + pb.inv_off + col * m;
    double *dst = X + pb.inv_off + col * m;
    double Rb[9];
#pragma unroll
    for (int k = 0; k < 9; ++k)
        Rb[k] = R[9 * pb.body + k];
    for (int r0 = 0; r0 < m; r0 += kPlaceRows) {
        const int rows = min(kPlaceRows, m - r0);
#pragma unroll
        for (int q = 0; q < 3; ++q)
            for (int i = t; i < rows; i += kPlaceThreads)
                tile[q][i] = src[(long long)q * m + r0 + i];
        __syncthreads();
        if (3 * t < rows) { // rows is a multiple of 3: the thread's tile is whole
            double x[3][3], y[3][3];
#pragma unroll
            for (int q = 0; q < 3; ++q)
#pragma unroll
                for (int p = 0; p < 3; ++p)
                    x[q][p] = tile[q][3 * t + p];
            rotate_tile(Rb, x, y);
#pragma unroll
            for (int q = 0; q < 3; ++q)
#pragma unroll
                for (int p = 0; p < 3; ++p)
                    tile[q][3 * t + p] = y[q][p];
        }
        __syncthreads();
#pragma unroll
        for (int q = 0; q < 3; ++q)
            for (int i = t; i < rows; i += kPlaceThreads)
                dst[(long long)q * m + r0 + i] = tile[q][i];
        __syncthreads();
    }
}

} // namespace skb

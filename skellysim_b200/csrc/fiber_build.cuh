// fiber_build.cuh -- the per-fiber operators of one timestep built on the device (skb_flow_build_fiber_operators).
//
//   fiber_assemble_kernel  A_ (4n x 4n), force_operator_ (3n x 4n) and xs_ of every fiber, column-major as Eigen stores
//                          them, from the node positions x_, length_ and the class matrices D_k_0 / P_downsample_bc:
//                          update_derivatives (fiber_finite_difference.cpp:62-68), update_linear_operator (:97-187),
//                          the operator half of apply_bc_rectangular (:347-512) and update_force_operator (:317-335).
//       One CTA per (fiber, tile of T columns).  The raw operator of update_linear_operator is a sum of row-scaled
//       derivative matrices, so every entry is formed where it is needed: the CTA writes its 4n x T slice of the raw
//       operator into shared memory, then rows [0, 4n-14) of A_ = P_downsample_bc * raw walk each row's non-zero column
//       range of the block-diagonal P (the exact zeros skipped change the summation order only), and the 14 boundary
//       rows are written from their formulas.
//   fiber_inverse_kernel   A_^-1 of every fiber (update_preconditioner, :340, then A_LU_.inverse()): in-place
//       Gauss-Jordan elimination with partial pivoting, the matrix in shared memory.  A cluster of `cs` CTAs holds one
//       matrix, every CTA a block of whole columns: cs = 1 for 4n <= 128 (n <= 32, 132 KB); larger n spread the
//       matrix over the cluster's distributed shared memory (n = 64: 3 CTAs, n = 128: 10).  Per pivot step the CTA that
//       owns the pivot column searches it, publishes the pivot row and the (row-swapped) column in its shared memory,
//       one cluster barrier later every CTA reads them and updates its own columns.  The column interchanges that
//       undo the pivoting are applied when the result is written out.
#pragma once
#include <cooperative_groups.h>
#include <cuda_runtime.h>

namespace skb {

constexpr int kBuildThreads = 256;    // fiber_assemble_kernel
constexpr int kInverseThreads = 512;  // fiber_inverse_kernel
constexpr int kBuildMinNodes = 8;     // the 8-point stencil of D_4 (finite_diff(alpha, 4, 8))
constexpr int kBuildMaxNodes = 128;   // fiber_finite_difference.cpp:522 allows up to 128
constexpr int kInverseMaxCluster = 16; // non-portable cluster size of sm_90
constexpr size_t kInverseSmemMax = 227 * 1024;

// matches skb_fiber_params of the C ABI (48 bytes)
struct FiberParamsDev {
    double length_prev, bending_rigidity, radius, penalty_param, beta_tstep;
    int minus_clamped, plus_hinged;
};

struct FiberItem {
    long long a_off, f_off; // element offsets of A_ / force_operator_ in op_A / op_F (the build only)
    long long node;         // first node of the fiber in r_fib (all fibers)
    long long own_node;     // first node among the own fibers (op_xs; the RHS's v, f and, times 4, its output)
    long long cls;          // element offset of the class block [D_1_0 | P_downsample_bc | D_2_0 | D_3_0 | D_4_0]
    long long rng;          // element offset of the class's P row ranges in the range buffer
    int n, fiber;           // nodes; index of the fiber in the container (fiber_length)
};

struct FiberTileItem {
    int item; // FiberItem index == params index
    int col0; // first column of the tile
};

// columns per assembly tile: the tile of the raw operator (4n x T) stays within 32 KB of shared memory
__host__ __device__ inline int build_tile_cols(int n) {
    const int t = 4096 / (4 * n);
    return t < 32 ? t : 32;
}
__host__ __device__ inline size_t build_smem_bytes(int n) {
    return ((size_t)4 * n * build_tile_cols(n) + (size_t)12 * n) * sizeof(double);
}

// columns per CTA and shared memory of fiber_inverse_kernel for an m x m matrix held by a cluster of cs CTAs
__host__ __device__ inline int inverse_cols(int m, int cs) { return (m + cs - 1) / cs; }
__host__ __device__ inline size_t inverse_smem_bytes(int m, int cs) {
    const int w = inverse_cols(m, cs);
    // matrix slice (leading dimension m + 1: odd, so that row accesses spread over the banks) | published pivot column
    // x 2 (double-buffered) | scaled pivot row | pivot of every step, its published copy x 2, column permutation
    return ((size_t)(m + 1) * w + 2 * (size_t)m + w) * sizeof(double) + ((size_t)2 * m + 2) * sizeof(int);
}
inline int inverse_cluster_size(int m) {
    for (int cs = 1; cs <= kInverseMaxCluster; ++cs)
        if (inverse_smem_bytes(m, cs) <= kInverseSmemMax)
            return cs;
    return 0;
}

// update_derivatives, K = 2 or 3: x_^{(k)} = (2 / length_prev_)^k x_ D_k_0 into d1 + 3n (k-1), [n x 3] each, k = 1 .. K
// (D_3_0 follows D_2_0).  Thread t forms the entries e = t (mod blockDim.x); the caller synchronises.  (ffd.cpp:62-68)
template <int K>
__device__ __forceinline__ void update_derivatives(const double *xv, const double *D1, const double *D2, int n,
                                                   double sp, double *d1) {
    const double *D3 = D2 + (size_t)n * n;
    double *d2 = d1 + 3 * n, *d3 = d2 + 3 * n;
    for (int e = threadIdx.x; e < 3 * n; e += blockDim.x) {
        const int i = e / 3, c = e - 3 * i;
        double s1 = 0.0, s2 = 0.0, s3 = 0.0;
        for (int j = 0; j < n; ++j) {
            const double xj = xv[3 * j + c];
            s1 = fma(D1[i * n + j], xj, s1);
            s2 = fma(D2[i * n + j], xj, s2);
            if (K == 3)
                s3 = fma(D3[i * n + j], xj, s3);
        }
        d1[e] = sp * s1;
        d2[e] = (sp * sp) * s2;
        if (K == 3)
            d3[e] = (sp * sp * sp) * s3;
    }
}

struct BuildArgs {
    const FiberItem *items;
    const FiberTileItem *tiles;
    const FiberParamsDev *params;
    const double *class_mats;
    const int2 *row_range;
    const double *r_fib;  // 3 x N_f, all fibers
    const double *length; // length_ of every fiber of the container
    double dt, eta;
    double *A, *F, *xs;   // op_A, op_F, op_xs
};

__global__ void __launch_bounds__(kBuildThreads) fiber_assemble_kernel(const BuildArgs a) {
    extern __shared__ double fb_smem[];
    const FiberTileItem tile = a.tiles[blockIdx.x];
    const FiberItem it = a.items[tile.item];
    const FiberParamsDev prm = a.params[tile.item];
    const int n = it.n, m = 4 * n, bc = m - 14, T = build_tile_cols(n);
    const int ncols = min(T, m - tile.col0);
    double *raw = fb_smem;                  // [m x T] column-major: the raw operator's columns of this tile
    double *xv = raw + (size_t)m * T;       // [n x 3] positions
    double *d1 = xv + 3 * n, *d2 = d1 + 3 * n, *d3 = d2 + 3 * n; // xs_, xss, xsss ([n x 3] each)
    const double *D1 = a.class_mats + it.cls;                 // pre-transposed: row i of D_k is D_k_0[i*n, i*n+n)
    const double *P = D1 + (size_t)n * n;
    const double *D2 = P + (size_t)bc * m, *D3 = D2 + (size_t)n * n, *D4 = D3 + (size_t)n * n;

    for (int e = threadIdx.x; e < 3 * n; e += blockDim.x)
        xv[e] = a.r_fib[3 * it.node + e];
    __syncthreads();
    update_derivatives<3>(xv, D1, D2, n, 2.0 / prm.length_prev, d1);
    __syncthreads();
    if (tile.col0 == 0)
        for (int e = threadIdx.x; e < 3 * n; e += blockDim.x)
            a.xs[3 * it.own_node + e] = d1[e];

    // update_constants (fiber_finite_difference.hpp:140-144); derivative matrices with length_ (ffd.cpp:101-104)
    const double L = a.length[it.fiber];
    const double eps = prm.radius / L;
    const double c0 = -log(M_E * (eps * eps)) / (8.0 * M_PI * a.eta), c1 = 2.0 / (8.0 * M_PI * a.eta);
    const double E = prm.bending_rigidity, bdt = prm.beta_tstep / a.dt;
    const double s1 = 2.0 / L, s2 = s1 * s1, s3 = s2 * s1, s4 = s2 * s2;

    // the raw operator of update_linear_operator (ffd.cpp:146-186) and force_operator_ (ffd.cpp:326-334) on this tile
    for (int e = threadIdx.x; e < m * ncols; e += blockDim.x) {
        const int R = e % m, cl = e / m, C = tile.col0 + cl;
        const int ra = R / n, i = R - ra * n, cb = C / n, j = C - cb * n;
        const double dlt = i == j ? 1.0 : 0.0;
        const double *xs = d1 + 3 * i, *xss = d2 + 3 * i;
        double v;
        if (ra < 3 && cb < 3) {
            const double D4ij = D4[i * n + j] * s4;
            if (ra == cb) {
                const double xa = xs[ra];
                v = (bdt * dlt + (E * c0) * (D4ij * (1.0 + xa * xa))) + (E * c1) * (D4ij * (1.0 - xa * xa));
            } else {
                v = (E * (c0 - c1)) * (D4ij * (xs[ra] * xs[cb]));
            }
        } else if (ra < 3) {
            v = -(c0 * 2.0) * ((D1[i * n + j] * s1) * xs[ra]) - (c0 + c1) * (dlt * xss[ra]);
        } else if (cb < 3) {
            v = (-(c1 + 7.0 * c0) * E) * ((D4[i * n + j] * s4) * xss[cb]) -
                ((6.0 * c0) * E) * ((D3[i * n + j] * s3) * d3[3 * i + cb]) -
                prm.penalty_param * ((D1[i * n + j] * s1) * xs[cb]);
        } else {
            const double q = (xss[0] * xss[0] + xss[1] * xss[1]) + xss[2] * xss[2];
            v = (-2.0 * c0) * (D2[i * n + j] * s2) + (c0 + c1) * (dlt * q);
        }
        raw[R + (size_t)cl * m] = v;
        if (R < 3 * n) { // force_operator_: -E D_4 on the diagonal blocks, diag(xss) + D_1 .* xs in the tension column
            double f = 0.0;
            if (cb == ra)
                f = -E * (D4[i * n + j] * s4);
            else if (cb == 3)
                f = dlt * xss[ra] + (D1[i * n + j] * s1) * xs[ra];
            a.F[it.f_off + R + (long long)C * (3 * n)] = f;
        }
    }
    __syncthreads();

    // rows [0, 4n-14): A_ = P_downsample_bc * raw over the non-zero columns of each row of P       (ffd.cpp:356)
    const int2 *rg = a.row_range + it.rng;
    for (int e = threadIdx.x; e < bc * ncols; e += blockDim.x) {
        const int r = e % bc, cl = e / bc;
        const int2 cr = rg[r];
        const double *col = raw + (size_t)cl * m;
        double acc = 0.0;
        for (int c = cr.x; c < cr.y; ++c)
            acc = fma(P[r + (size_t)c * bc], col[c], acc);
        a.A[it.a_off + r + (long long)(tile.col0 + cl) * m] = acc;
    }
    // the 14 boundary rows                                                                          (ffd.cpp:362-512)
    const int e_ = n - 1;
    const double *xs0 = d1, *xss0 = d2, *xse = d1 + 3 * e_, *xsse = d2 + 3 * e_;
    for (int e = threadIdx.x; e < 14 * ncols; e += blockDim.x) {
        const int t = e % 14, C = tile.col0 + e / 14;
        const int cb = C / n, j = C - cb * n;
        double v = 0.0;
        if (t < 4) { // minus end, first condition
            if (prm.minus_clamped) { // Velocity                                                     (ffd.cpp:366-384)
                if (t < 3)
                    v = C == t * n ? bdt : 0.0;
                else
                    v = cb < 3 ? ((6.0 * E * c0) * xss0[cb]) * (D3[j] * s3) : (2.0 * c0) * (D1[j] * s1);
            } else { // Force                                                                        (ffd.cpp:386-405)
                if (t < 3)
                    v = cb == t ? E * (D3[j] * s3) : (C == 3 * n ? -xs0[t] : 0.0);
                else
                    v = cb < 3 ? (-E * (D2[j] * s2)) * xss0[cb] : (C == 3 * n ? -1.0 : 0.0);
            }
        } else if (t < 7) { // minus end, second condition: AngularVelocity or Torque                (ffd.cpp:415-433)
            if (cb == t - 4)
                v = prm.minus_clamped ? bdt * (D1[j] * s1) : D2[j] * s2;
        } else if (t < 11) { // plus end, first condition
            if (prm.plus_hinged) { // Velocity                                                       (ffd.cpp:443-464)
                if (t < 10)
                    v = C == (t - 6) * n - 1 ? bdt : 0.0;
                else
                    v = cb < 3 ? (6.0 * E * c0) * (D3[e_ * n + j] * s3) * xsse[cb] : (2.0 * c0) * (D1[e_ * n + j] * s1);
            } else { // Force                                                                        (ffd.cpp:466-487)
                if (t < 10)
                    v = cb == t - 7 ? -E * (D3[e_ * n + j] * s3) : (C == m - 1 ? xse[t - 7] : 0.0);
                else
                    v = cb < 3 ? (E * (D2[e_ * n + j] * s2)) * xsse[cb] : (C == m - 1 ? 1.0 : 0.0);
            }
        } else if (cb == t - 11) { // plus end Torque                                                (ffd.cpp:497-505)
            v = D2[e_ * n + j] * s2;
        }
        a.A[it.a_off + bc + t + (long long)C * m] = v;
    }
}

// In-place Gauss-Jordan inverse of one m x m matrix per cluster (see the top of the file).  Launched per node count
// with cluster dimension cs; a_off[blockIdx.x / cs] is the matrix of the cluster in A (read) and Ainv (written).
// Every lane keeps its rows of the pivot column in registers: QMAX >= m / 32.
template <int QMAX>
__global__ void __launch_bounds__(kInverseThreads) fiber_inverse_kernel(const long long *__restrict__ a_off,
                                                                        const double *__restrict__ A,
                                                                        double *__restrict__ Ainv, int m) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    extern __shared__ double fi_smem[];
    const int cs = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
    const int w = inverse_cols(m, cs), ld = m + 1;
    const int c0 = rank * w, wl = min(w, m - c0);
    double *Al = fi_smem;                    // [ld x w]: columns [c0, c0 + wl) of the matrix
    double *pcol = Al + (size_t)ld * w;      // [2][m] published pivot column (owner of the step's column)
    double *rowv = pcol + 2 * m;             // [w] the scaled pivot row, own columns
    int *piv = reinterpret_cast<int *>(rowv + w); // [m] pivot row of every step
    int *perm = piv + m;                     // [m] final column permutation
    int *ppub = perm + m;                    // [2] published pivot row
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const long long off = a_off[blockIdx.x / cs];

    for (int jl = warp; jl < wl; jl += nwarps)
        for (int i = lane; i < m; i += 32)
            Al[i + jl * ld] = A[off + i + (long long)(c0 + jl) * m];
    __syncthreads();

    for (int k = 0; k < m; ++k) {
        const int owner = k / w, buf = k & 1;
        if (rank == owner) {
            const double *col = Al + (k - c0) * ld;
            if (warp == 0) { // partial pivoting: the first row of largest magnitude in rows [k, m)
                double bv = -1.0;
                int bi = k;
                for (int i = k + lane; i < m; i += 32) {
                    const double v = fabs(col[i]);
                    if (v > bv) {
                        bv = v;
                        bi = i;
                    }
                }
                for (int o = 16; o > 0; o >>= 1) {
                    const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
                    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                    if (ov > bv || (ov == bv && oi < bi)) {
                        bv = ov;
                        bi = oi;
                    }
                }
                if (lane == 0)
                    ppub[buf] = bi;
            }
            __syncthreads();
            const int p = ppub[buf];
            for (int i = threadIdx.x; i < m; i += blockDim.x)
                pcol[buf * m + i] = col[i == k ? p : (i == p ? k : i)];
        }
        // the owner's pivot column is published; the buffer it wrote is not written again before every CTA has passed
        // the next step's barrier, so one barrier per step suffices
        cluster.sync();
        const double *rc = cluster.map_shared_rank(pcol, owner) + buf * m;
        const int p = *cluster.map_shared_rank(ppub + buf, owner);
        const double inv = 1.0 / rc[k];
        if (threadIdx.x == 0)
            piv[k] = p;
        for (int jl = threadIdx.x; jl < wl; jl += blockDim.x) { // row interchange and scaled pivot row
            double *col = Al + jl * ld;
            double ak = col[k];
            if (p != k) {
                const double ap = col[p];
                col[p] = ak;
                ak = ap;
            }
            const double r = c0 + jl == k ? inv : ak * inv;
            rowv[jl] = r;
            col[k] = r;
        }
        double cv[QMAX];
#pragma unroll
        for (int q = 0; q < QMAX; ++q) {
            const int i = lane + 32 * q;
            cv[q] = i < m ? rc[i] : 0.0;
        }
        __syncthreads();
        for (int jl = warp; jl < wl; jl += nwarps) { // eliminate column k from every other row
            double *col = Al + jl * ld;
            const double r = rowv[jl];
            const bool pivot_col = c0 + jl == k;
#pragma unroll
            for (int q = 0; q < QMAX; ++q) {
                const int i = lane + 32 * q;
                if (i < m && i != k)
                    col[i] = fma(-cv[q], r, pivot_col ? 0.0 : col[i]);
            }
        }
        __syncthreads();
    }
    // undo the pivoting: the column interchanges (k, piv[k]) in reverse order, as a permutation of the output columns
    if (threadIdx.x == 0) {
        for (int c = 0; c < m; ++c)
            perm[c] = c;
        for (int k = m - 1; k >= 0; --k) {
            const int t = perm[k];
            perm[k] = perm[piv[k]];
            perm[piv[k]] = t;
        }
        for (int c = 0; c < m; ++c) // output column of every elimination column
            piv[perm[c]] = c;
    }
    __syncthreads();
    for (int jl = warp; jl < wl; jl += nwarps) {
        const long long dst = off + (long long)piv[c0 + jl] * m;
        for (int i = lane; i < m; i += 32)
            Ainv[dst + i] = Al[i + jl * ld];
    }
    cluster.sync(); // no CTA leaves while another may still read its published column
}

} // namespace skb

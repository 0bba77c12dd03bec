// fiber_ops.cuh -- per-fiber dense operators of the GMRES matvec, device resident (SURVEY.md §8f N2).
//
//   fiber_gemv_kernel<MODE>   y_f = M_f x_f for every fiber f; M_f column-major as Eigen stores
//                             FiberFiniteDifference::A_ (4n x 4n) and ::force_operator_ (3n x 4n).  HBM-bound: every
//                             matrix element is read once per matvec, 8 B / FMA.
//       MODE 0  out[row] = (M x)[row]                                  (A_^-1 x: the fiber preconditioner)
//       MODE 1  force layout of FiberContainerFiniteDifference::apply_fiber_force (fcfd.cpp:272-287)
//       MODE 2  the whole of FiberFiniteDifference::matvec (src/core/fiber_finite_difference.cpp:276-312) in ONE pass:
//               res = A_ x - P_downsample_bc vT(v) + xs_vT + y_BC -- the velocity / boundary part rides on the
//               HBM-bound GEMV instead of a second launch that re-reads and re-writes res.
//
// Work decomposition: one CTA of 256 threads per (fiber, 32-row block); thread (lr, q) accumulates row row0+lr over the
// columns j == q (mod 8); a warp reads 32 consecutive rows of one column = 256 contiguous bytes.  32-row blocks tile
// both operator heights (3n and 4n are multiples of 32 for every allowed n >= 32, fiber_finite_difference.cpp:522),
// so no CTA is half empty.
#pragma once
#include <cuda_runtime.h>

namespace skb {

constexpr int kFiberGemvRows = 32;   // rows per CTA
constexpr int kFiberGemvSlices = 8;  // column slices per row
constexpr int kFiberGemvThreads = kFiberGemvRows * kFiberGemvSlices;
constexpr size_t kFiberGemvSmemMax = 200 * 1024; // dynamic shared memory the kernels are allowed (prepare_fiber_kernels)

struct FiberGemvItem {
    long long mat_off; // element offset of M_f in the concatenated operator buffer
    long long x_off;   // element offset of x_f (4 * node offset)
    long long out_off; // MODE 0/2: element offset of y_f;  MODE 1: node offset of the fiber
    int rows, cols;    // shape of M_f
    int row0;          // first row of this CTA
    int n_nodes;       // nodes of the fiber
    int fiber, pad;    // index of the fiber among the resident ones (MODE 2: xs / length_prev / class / v_boundary)
};

// everything MODE 2 needs beyond the GEMV operands; the fiber-indexed arrays start at the first resident fiber
struct FiberVelArgs {
    const double *xs;          // [N_own*3] tangents xs_
    const double *v;           // [N_own*3] velocities at the fiber nodes
    const double *length_prev; // [n_fibers]
    const int *plus_velocity;  // [n_fibers] bc_plus_.first == Velocity
    const double *class_mats;  // D_1_0 (n x n) and P_downsample_bc ((4n-14) x 4n) of every node count, column-major
    const long long *class_D;  // [n_fibers] element offset of the fiber's D_1_0 in class_mats
    const long long *class_P;  // [n_fibers] ... of its P_downsample_bc
    const int2 *row_range;     // per class: [4n-14] first / one-past-last non-zero column of every row of P, then [n]
                               // first / one-past-last non-zero row of every column of D_1_0 (banded: 5-point stencils)
    const long long *class_R;  // [n_fibers] element offset of the fiber's ranges
    const double *v_boundary;  // [n_fibers*7] or nullptr
};

// CTAs per SM the register budget must allow: the kernels are latency x bandwidth bound (8 loads in flight per thread),
// so resident CTAs are what counts (8 x 256 threads x 32 registers fill the register file).
template <int MODE>
__global__ void __launch_bounds__(kFiberGemvThreads, 8)
    fiber_gemv_kernel(const FiberGemvItem *__restrict__ items, const double *__restrict__ mats,
                      const double *__restrict__ x, double *__restrict__ out, const FiberVelArgs va) {
    extern __shared__ double fg_smem[];
    const FiberGemvItem &it = items[blockIdx.x]; // (fields are re-read where needed: L1-resident, and 12 registers less)
    const int colsp = (it.cols + 1) & ~1;
    double *xs_sh = fg_smem;             // cols
    double *part = fg_smem + colsp;      // kFiberGemvSlices x kFiberGemvRows
    double *vT = part + kFiberGemvThreads; // MODE 2: 4n
    double *s_sh = vT + colsp;             // MODE 2: n
    for (int j = threadIdx.x; j < it.cols; j += kFiberGemvThreads)
        xs_sh[j] = x[it.x_off + j];
    const int n = it.n_nodes;
    // MODE 0/1: the first eight columns of this thread's row go out to HBM NOW, ahead of the x load.  MODE 2 does not
    // prefetch them ahead of its preamble: the eight live values pushed it to 62 registers = 4 CTAs per SM; without them
    // it fits 32 registers = 8 CTAs per SM, and the other CTAs' loads cover this CTA's preamble better than its own early
    // loads do (a cp.async prefetch into shared memory was slower than both).
    constexpr bool kPre = MODE != 2;
    const int lr0 = threadIdx.x & (kFiberGemvRows - 1), q0 = threadIdx.x / kFiberGemvRows;
    const bool row_ok = it.row0 + lr0 < it.rows;
    const bool first_ok = kPre && row_ok && q0 + 7 * kFiberGemvSlices < it.cols;
    double v0[8];
    if (kPre && first_ok) {
        const double *m0 = mats + it.mat_off + it.row0 + lr0;
#pragma unroll
        for (int u = 0; u < 8; ++u)
            v0[u] = __ldg(m0 + (long long)(q0 + u * kFiberGemvSlices) * it.rows);
    }
    int2 my_rg = make_int2(0, 0);
    if (MODE == 2) {
        // Which entries of vT = [v_x; v_y; v_z; D_1^T (xs . v)] (ffd.cpp:280-293) do this CTA's rows of P touch?  P is
        // block diagonal, so a 32-row block needs one or two of the four segments -- and D_1^T s only for the last.
        __shared__ int c_lo, c_hi;
        if (threadIdx.x == 0) {
            c_lo = 4 * n;
            c_hi = 0;
        }
        __syncthreads();
        const int bc = 4 * n - 14, row_t = it.row0 + (int)threadIdx.x;
        if (threadIdx.x < kFiberGemvRows && row_t < bc) {
            my_rg = va.row_range[va.class_R[it.fiber] + row_t];
            if (my_rg.y > my_rg.x) {
                atomicMin(&c_lo, my_rg.x);
                atomicMax(&c_hi, my_rg.y);
            }
        }
        __syncthreads();
        const int lo = c_lo, hi = c_hi;
        const long long node_off = it.x_off / 4;
        const double *xt = va.xs + 3 * node_off, *v = va.v + 3 * node_off;
        const bool need_D = hi > 3 * n;
        for (int i = threadIdx.x; i < n; i += kFiberGemvThreads) {
            const double vx = v[3 * i], vy = v[3 * i + 1], vz = v[3 * i + 2];
            vT[i] = vx;
            vT[n + i] = vy;
            vT[2 * n + i] = vz;
            if (need_D)
                s_sh[i] = xt[3 * i] * vx + xt[3 * i + 1] * vy + xt[3 * i + 2] * vz;
        }
        if (need_D) {
            __syncthreads();
            // (D_1^T s)[j] = sum_i D_1(i, j) s_i over the non-zero rows of column j, D_1 = D_1_0 * 2 / length_prev
            const double scale = 2.0 / va.length_prev[it.fiber];
            const double *D = va.class_mats + va.class_D[it.fiber];
            const int2 *col_rg = va.row_range + va.class_R[it.fiber] + bc;
            for (int j = threadIdx.x; j < n; j += kFiberGemvThreads) {
                const int2 rg = col_rg[j];
                const double *col = D + (long long)j * n;
                double acc = 0.0;
                for (int i = rg.x; i < rg.y; ++i)
                    acc = fma(col[i], s_sh[i], acc);
                vT[3 * n + j] = scale * acc;
            }
        }
        (void)lo;
    }
    __syncthreads();
    const int lr = threadIdx.x & (kFiberGemvRows - 1), q = threadIdx.x / kFiberGemvRows;
    const int row = it.row0 + lr;
    double acc = 0.0;
    if (row < it.rows) {
        const double *m = mats + it.mat_off + row;
        const long long ld = it.rows;
        int j = q;
        if (kPre && first_ok) { // (loaded before the preamble)
#pragma unroll
            for (int u = 0; u < 8; ++u)
                acc = fma(v0[u], xs_sh[j + u * kFiberGemvSlices], acc);
            j += 8 * kFiberGemvSlices;
        }

        // 8 independent loads in flight per thread
        for (; j + 7 * kFiberGemvSlices < it.cols; j += 8 * kFiberGemvSlices) {
            double v[8];
#pragma unroll
            for (int u = 0; u < 8; ++u)
                v[u] = __ldg(m + (long long)(j + u * kFiberGemvSlices) * ld);
#pragma unroll
            for (int u = 0; u < 8; ++u)
                acc = fma(v[u], xs_sh[j + u * kFiberGemvSlices], acc);
        }
        for (; j < it.cols; j += kFiberGemvSlices)
            acc = fma(__ldg(m + (long long)j * ld), xs_sh[j], acc);
        if (MODE == 2) {
            // - (P_downsample_bc vT)[row] for row < 4n-14, over the row's non-zero columns only: P is block diagonal in
            // the reference (three (n-4) x n blocks and one (n-2) x n, ffd.cpp:551-555), 75 % structural zeros
            const int bc = 4 * n - 14;
            if (row < bc) {
                const int2 rg = va.row_range[va.class_R[it.fiber] + row]; // (L1-resident: read by the 8 slices of a row)
                const double *p = va.class_mats + va.class_P[it.fiber] + row;
                double a2 = 0.0;
                for (int c = rg.x + q; c < rg.y; c += kFiberGemvSlices)
                    a2 = fma(__ldg(p + (long long)c * bc), vT[c], a2);
                acc -= a2;
            }
        }
    }
    part[q * kFiberGemvRows + lr] = acc;
    __syncthreads();
    if (q == 0 && row < it.rows) {
        double s = part[lr];
#pragma unroll
        for (int u = 1; u < kFiberGemvSlices; ++u)
            s += part[u * kFiberGemvRows + lr];
        if (MODE == 1) {
            const int k = row / n, i = row - k * n;
            out[3 * (it.out_off + i) + k] = s;
        } else {
            if (MODE == 2) {
                // the 14 boundary rows: xs_vT and y_BC                                     (ffd.cpp:298-309)
                const int t = row - (4 * n - 14);
                if (t >= 0) {
                    const long long node_off = it.x_off / 4;
                    const double *xt = va.xs + 3 * node_off, *v = va.v + 3 * node_off;
                    if (t == 3)
                        s += v[0] * xt[0] + v[1] * xt[1] + v[2] * xt[2];
                    if (va.v_boundary && t < 7)
                        s += va.v_boundary[7 * (long long)it.fiber + t];
                    if (t == 10 && va.plus_velocity[it.fiber]) {
                        const int e = 3 * (n - 1);
                        s += v[e] * xt[e] + v[e + 1] * xt[e + 1] + v[e + 2] * xt[e + 2];
                    }
                }
            }
            out[it.out_off + row] = s;
        }
    }
}

} // namespace skb

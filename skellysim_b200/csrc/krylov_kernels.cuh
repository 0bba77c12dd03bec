// krylov_kernels.cuh -- the vector passes of right-preconditioned restarted GMRES (skb_solve.cu, the only includer).
//
// The Krylov basis V is column-major with leading dimension ld (n rounded up to 32 rows); column j starts at V + j ld.
// Every pass splits the n rows into one contiguous row block per CTA (KrylovGrid: fixed by n and the device's SM count)
// and walks its block in tiles of 32 rows, one row per lane.  A dot product is summed in a fixed order: inside a tile a
// warp's shuffle tree, over the tiles of a block in tile order into a shared accumulator, and over the blocks in block
// order by krylov_combine_kernel.  No atomics: a solve is bitwise reproducible run to run.
//
// One Arnoldi step with w = A P^-1 v_k stored in column k + 1 (ICGS: two classical Gram-Schmidt passes) is three
// passes over the k + 1 columns of V:
//   A  (kDots):       h1 = V^T w, and w^T w                                  reads V and w
//   B  (kUpdateDots): w -= V h1, then h2 = V^T w of the updated rows         reads V, reads and writes w
//   C  (kUpdateNorm): w -= V h2, then w^T w                                  reads V, reads and writes w
// Pass B's second use of a tile of V follows its first at once: the tile (32 rows x k columns, 77 KB at k = 300) is
// still in L1 / L2, so each pass reads V from HBM once: 3 x 8 k n bytes per step, plus O(n) for w.
#pragma once
#include <cuda_runtime.h>

namespace skb {

constexpr int kKrylovThreads = 256; // 8 warps; a tile is 32 rows
constexpr int kKrylovWarps = kKrylovThreads / 32;

enum KrylovPass { kDots = 0, kUpdateDots = 1, kUpdateNorm = 2 };

// Per CTA: w[r] -= sum_j V[r, j] coef[j] (kUpdate*), then part[blockIdx.x * ldp + j] = its rows' share of
// V[:, j]^T w for j < k, and of w^T w at index k (kDots) or 0 (kUpdateNorm).  Dynamic shared memory:
// (2 k + 1) doubles for coef and the accumulators, plus 32 (the tile of w) + 8 x 32 (the warps' partial row sums).
template <int PASS>
__global__ void __launch_bounds__(kKrylovThreads) krylov_pass_kernel(const double *__restrict__ V, long long ld, int k,
                                                                      double *__restrict__ w,
                                                                      const double *__restrict__ coef, long long n,
                                                                      long long rows_per, double *__restrict__ part,
                                                                      int ldp) {
    extern __shared__ double sm[];
    double *c = sm;                 // [k]   coefficients of the update
    double *acc = c + k;            // [k+1] this CTA's dot accumulators
    double *wt = acc + k + 1;       // [32]  the tile of w
    double *red = wt + 32;          // [8][32] partial row sums of the update
    const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
    constexpr bool update = PASS != kDots;
    for (int j = threadIdx.x; j < k; j += kKrylovThreads) {
        if (update)
            c[j] = coef[j];
        acc[j] = 0.0;
    }
    if (threadIdx.x == 0)
        acc[k] = 0.0;
    __syncthreads();
    const long long r0 = (long long)blockIdx.x * rows_per;
    const long long r1 = min(n, r0 + rows_per);
    for (long long t0 = r0; t0 < r1; t0 += 32) {
        const long long r = t0 + lane;
        const bool live = r < r1;
        if (update) {
            double s = 0.0;
#pragma unroll 4
            for (int j = wp; j < k; j += kKrylovWarps)
                s += live ? V[j * ld + r] * c[j] : 0.0;
            red[wp * 32 + lane] = s;
            __syncthreads();
            if (wp == 0) {
                double tot = red[lane];
#pragma unroll
                for (int q = 1; q < kKrylovWarps; ++q)
                    tot += red[q * 32 + lane];
                const double wn = live ? w[r] - tot : 0.0;
                if (live)
                    w[r] = wn;
                wt[lane] = wn;
            }
        } else if (wp == 0) {
            wt[lane] = live ? w[r] : 0.0;
        }
        __syncthreads();
        const double wl = wt[lane];
        if (PASS != kUpdateNorm) {
#pragma unroll 4
            for (int j = wp; j < k; j += kKrylovWarps) {
                double p = live ? V[j * ld + r] * wl : 0.0;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1)
                    p += __shfl_down_sync(0xffffffffu, p, o);
                if (lane == 0)
                    acc[j] += p;
            }
        }
        if (PASS != kUpdateDots && wp == 0) { // w^T w: warp 0 owns index k (kDots) or 0 (kUpdateNorm)
            double p = wl * wl;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1)
                p += __shfl_down_sync(0xffffffffu, p, o);
            if (lane == 0)
                acc[PASS == kDots ? k : 0] += p;
        }
        __syncthreads(); // wt and red are rewritten by the next tile
    }
    const int m = PASS == kDots ? k + 1 : (PASS == kUpdateDots ? k : 1);
    for (int j = threadIdx.x; j < m; j += kKrylovThreads)
        part[(long long)blockIdx.x * ldp + j] = acc[j];
}

// out[j] = sum over the CTAs c = 0 .. n_parts-1 of part[c * ldp + j], one CTA per j: thread t sums c = t, t + 128, ...
// in order, then a fixed tree over the threads
constexpr int kCombineThreads = 128;
__global__ void __launch_bounds__(kCombineThreads) krylov_combine_kernel(const double *__restrict__ part, int n_parts,
                                                                          int ldp, double *__restrict__ out) {
    __shared__ double s[kCombineThreads];
    const int j = blockIdx.x;
    double a = 0.0;
    for (int c = threadIdx.x; c < n_parts; c += kCombineThreads)
        a += part[(long long)c * ldp + j];
    s[threadIdx.x] = a;
    __syncthreads();
    for (int h = kCombineThreads / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h)
            s[threadIdx.x] += s[threadIdx.x + h];
        __syncthreads();
    }
    if (threadIdx.x == 0)
        out[j] = s[0];
}

// out = b - ax (ax == nullptr: out = b), and per CTA its rows' share of out^T out into part[blockIdx.x * ldp]
__global__ void __launch_bounds__(kKrylovThreads) krylov_residual_kernel(const double *__restrict__ b,
                                                                          const double *__restrict__ ax,
                                                                          double *__restrict__ out, long long n,
                                                                          long long rows_per, double *__restrict__ part,
                                                                          int ldp) {
    __shared__ double s[kKrylovThreads];
    const long long r0 = (long long)blockIdx.x * rows_per;
    const long long r1 = min(n, r0 + rows_per);
    double a = 0.0;
    for (long long r = r0 + threadIdx.x; r < r1; r += kKrylovThreads) {
        const double v = ax ? b[r] - ax[r] : b[r];
        out[r] = v;
        a += v * v;
    }
    s[threadIdx.x] = a;
    __syncthreads();
    for (int h = kKrylovThreads / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h)
            s[threadIdx.x] += s[threadIdx.x + h];
        __syncthreads();
    }
    if (threadIdx.x == 0)
        part[(long long)blockIdx.x * ldp] = s[0];
}

// v[r] /= sqrt(*nrm2): the next basis vector (the host has read the same *nrm2 and decided there is no breakdown)
__global__ void krylov_scale_kernel(double *__restrict__ v, long long n, const double *__restrict__ nrm2) {
    const double beta = sqrt(*nrm2);
    for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < n; r += (long long)gridDim.x * blockDim.x)
        v[r] /= beta;
}

// u = V[:, 0..k) y, y from device memory; one row per thread, the columns in order
__global__ void __launch_bounds__(kKrylovThreads) krylov_gemv_kernel(const double *__restrict__ V, long long ld, int k,
                                                                      const double *__restrict__ y,
                                                                      double *__restrict__ u, long long n) {
    extern __shared__ double ys[];
    for (int j = threadIdx.x; j < k; j += blockDim.x)
        ys[j] = y[j];
    __syncthreads();
    for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < n; r += (long long)gridDim.x * blockDim.x) {
        double s = 0.0;
        for (int j = 0; j < k; ++j)
            s += V[j * ld + r] * ys[j];
        u[r] = s;
    }
}

// x += z
__global__ void krylov_axpy_kernel(double *__restrict__ x, const double *__restrict__ z, long long n) {
    for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < n; r += (long long)gridDim.x * blockDim.x)
        x[r] += z[r];
}

} // namespace skb
